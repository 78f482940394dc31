"""Host restatement of the voxel-model operators (pcgb_hex_fill_field, pcgb_mg_create_field): the oracle of their tests.

A voxel box carries one Young's modulus per element; element e (x fastest) has the matrix Ck_e Ke with Ck_e = E_e h.  The
multigrid's coarse element matrices are element-level Galerkin products: coarse element (X, Y, Z) has the children
(2X + cx, 2Y + cy, 2Z + cz), c = cx + 2 cy + 4 cz, and

    K_E = sum_c Q_c^T K_child(c) Q_c,

Q_c the 24x24 trilinear interpolation from the coarse element's corners onto child c's nodes.  Every level here is an explicit
scipy matrix assembled from its element matrices (clamped x = 0 nodes dropped), so it can be checked against P^T A P with
gmg_cases.prolongation_matrix, and the V-cycle is gmg_cases.HostMultigrid's on those matrices.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import gmg_cases as G
from tests.gmg_cases import cheb_coeffs, lanczos_lambda, levels_of, prolongation_matrix, restrict  # noqa: F401


def child_weight(c, l, k):
    """Weight of coarse corner k on child c's local node l: prod_a phi_{k_a}(p_a), p = c + bits(l), phi_0 = (2-p)/2, phi_1 = p/2."""
    w = 1.0
    for a in range(3):
        p = ((c >> a) & 1) + ((l >> a) & 1)
        w *= 0.5 * p if (k >> a) & 1 else 0.5 * (2 - p)
    return w


def child_Q(c):
    """Q_c (24 x 24, child dofs x coarse dofs; dof = 3 node + dir)."""
    Q = np.zeros((24, 24))
    for l in range(8):
        for k in range(8):
            for d in range(3):
                Q[3 * l + d, 3 * k + d] = child_weight(c, l, k)
    return Q


Q = np.stack([child_Q(c) for c in range(8)])


def fine_elements(field, h, ke):
    """(nz, ny, nx, 24, 24): Ck_e Ke per element of the field (shape (nz, ny, nx)), Ck = E h."""
    return (np.asarray(field, dtype=np.float64) * h)[..., None, None] * ke


def galerkin(kf):
    """Coarse element matrices (nz/2, ny/2, nx/2, 24, 24) of fine ones (nz, ny, nx, 24, 24): sum_c Q_c^T K_child(c) Q_c."""
    out = 0.0
    for c in range(8):
        cx, cy, cz = c & 1, (c >> 1) & 1, c >> 2
        out = out + Q[c].T @ kf[cz::2, cy::2, cx::2] @ Q[c]
    return out


def assemble(kel, ng, e0=(0, 0, 0)):
    """Clamped sub-assembly of per-element matrices kel (nz, ny, nx, 24, 24) of the box at e0 in a mesh of ng elements, in the
    free-dof numbering of R.hex_box_csr (x fastest; nodes with global x index 0 dropped)."""
    nz, ny, nx = kel.shape[:3]
    x_lo = 1 if e0[0] == 0 else 0
    nxf = nx + 1 - x_lo
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex, ey, ez = ex.ravel(), ey.ravel(), ez.ravel()
    dofs = np.empty((ex.size, 24), dtype=np.int64)
    valid = np.empty((ex.size, 24), dtype=bool)
    for l in range(8):
        lx, ly, lz = ex + (l & 1), ey + ((l >> 1) & 1), ez + ((l >> 2) & 1)
        for d in range(3):
            dofs[:, 3 * l + d] = 3 * ((lz * (ny + 1) + ly) * nxf + (lx - x_lo)) + d
            valid[:, 3 * l + d] = lx >= x_lo
    rows = np.repeat(dofs[:, :, None], 24, axis=2)
    cols = np.repeat(dofs[:, None, :], 24, axis=1)
    ok = valid[:, :, None] & valid[:, None, :]
    vals = kel.reshape(-1, 24, 24)
    n = 3 * nxf * (ny + 1) * (nz + 1)
    A = sp.coo_matrix((vals[ok], (rows[ok], cols[ok])), shape=(n, n)).tocsr()
    A.sum_duplicates()
    A.sort_indices()
    return A


def field_csr(field, h, nu=0.3, ng=None, e0=(0, 0, 0)):
    """The fine voxel matrix of a box (field of the box's elements) with R.hex_ke."""
    return assemble(fine_elements(field, h, R.hex_ke(1.0, nu)), ng, e0)


def level_elements(field, h, nu=0.3, ke=None):
    """Element matrices of every level of the whole-box hierarchy: [fine, Galerkin level 1, level 2, ...]."""
    ke = R.hex_ke(1.0, nu) if ke is None else ke
    ne = tuple(int(v) for v in reversed(field.shape))
    out = [fine_elements(field, h, ke)]
    for _ in levels_of(ne)[1:]:
        out.append(galerkin(out[-1]))
    return out


def level_matrices(field, h, nu=0.3):
    """Scipy CSR of every level of the whole-box hierarchy (fine, then the Galerkin levels)."""
    return [assemble(k, None) for k in level_elements(field, h, nu)]


def assemble_ld(kel, e0=(0, 0, 0)):
    """The assembly of `assemble` in long double, as COO sorted by (row, col): rows, cols, values, sum of |terms| and the
    number of terms per entry (the rounding bound of a device sum of the same terms)."""
    nz, ny, nx = kel.shape[:3]
    x_lo = 1 if e0[0] == 0 else 0
    nxf = nx + 1 - x_lo
    n = 3 * nxf * (ny + 1) * (nz + 1)
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex, ey, ez = ex.ravel(), ey.ravel(), ez.ravel()
    dofs = np.empty((ex.size, 24), dtype=np.int64)
    valid = np.empty((ex.size, 24), dtype=bool)
    for l in range(8):
        lx, ly, lz = ex + (l & 1), ey + ((l >> 1) & 1), ez + ((l >> 2) & 1)
        for d in range(3):
            dofs[:, 3 * l + d] = 3 * ((lz * (ny + 1) + ly) * nxf + (lx - x_lo)) + d
            valid[:, 3 * l + d] = lx >= x_lo
    ok = valid[:, :, None] & valid[:, None, :]
    key = (dofs[:, :, None] * n + dofs[:, None, :])[ok]
    vals = np.asarray(kel, dtype=np.longdouble).reshape(-1, 24, 24)[ok]
    order = np.argsort(key, kind="stable")
    key, vals = key[order], vals[order]
    uk, start, count = np.unique(key, return_index=True, return_counts=True)
    return uk // n, uk % n, np.add.reduceat(vals, start), np.add.reduceat(np.abs(vals), start), count


def field_entries_ld(field, h, ke, rows, cols, x_lo=1):
    """Entries (rows[i], cols[i]) of the fine voxel matrix of a whole box (field shape (nz, ny, nx); free numbering with
    x_lo clamped planes dropped) in long double, without assembling it: sum over the <= 8 elements holding both nodes of
    Ck_e Ke[3 la + d, 3 lb + c].  Returns values, sum of |terms| and the number of terms per entry."""
    nz, ny, nx = field.shape
    nxf = nx + 1 - x_lo

    def node(i):
        nd = i // 3
        return nd % nxf + x_lo, (nd // nxf) % (ny + 1), nd // (nxf * (ny + 1)), i % 3

    ax, ay, az, d = node(np.asarray(rows, dtype=np.int64))
    bx, by, bz, c = node(np.asarray(cols, dtype=np.int64))
    ck = np.asarray(field, dtype=np.longdouble) * np.longdouble(h)
    kel = np.asarray(ke, dtype=np.longdouble)
    val = np.zeros(ax.size, dtype=np.longdouble)
    mag = np.zeros_like(val)
    cnt = np.zeros(ax.size, dtype=np.int64)
    for la in range(8):
        ox, oy, oz = ax - (la & 1), ay - ((la >> 1) & 1), az - (la >> 2)
        lbx, lby, lbz = bx - ox, by - oy, bz - oz
        ok = (ox >= 0) & (ox < nx) & (oy >= 0) & (oy < ny) & (oz >= 0) & (oz < nz)
        ok &= (lbx >= 0) & (lbx <= 1) & (lby >= 0) & (lby <= 1) & (lbz >= 0) & (lbz <= 1)
        lb = lbx + 2 * lby + 4 * lbz
        t = ck[np.where(ok, oz, 0), np.where(ok, oy, 0), np.where(ok, ox, 0)] * kel[3 * la + d, 3 * np.where(ok, lb, 0) + c]
        t = np.where(ok, t, 0)
        val += t
        mag += np.abs(t)
        cnt += ok
    return val, mag, cnt


class MatOp:
    """A scipy matrix with the interface gmg_cases' restatement uses (n, diag, @)."""

    def __init__(self, A):
        self.A = sp.csr_matrix(A)
        self.n = self.A.shape[0]
        self.diag = self.A.diagonal()

    def __matmul__(self, v):
        return self.A @ v


class HostFieldMultigrid(G.HostMultigrid):
    """gmg_cases.HostMultigrid's V-cycle on the Galerkin levels of a field: same smoother, Lanczos estimate, transfers and
    dense coarsest solve; only the level matrices differ.  lambdas / minv: as in HostMultigrid."""

    def __init__(self, field, h, degree=2, lo=0.25, lambdas=None, minv=None, nu=0.3, mats=None):
        ne = tuple(int(v) for v in reversed(field.shape))
        self.ne = levels_of(ne)
        self.degree, self.lo = degree, lo
        mats = level_matrices(field, h, nu) if mats is None else mats
        self.mats = mats
        self.A = [MatOp(A) for A in mats]
        self.dinv = [1.0 / A.diag for A in self.A]
        if minv is not None:
            self.dinv[0] = minv
        L = len(self.ne)
        self.lam = list(lambdas[:L - 1]) if lambdas is not None else [lanczos_lambda(self.A[l], self.dinv[l]) for l in range(L - 1)]
        self.coef = [cheb_coeffs(lam, degree, lo) for lam in self.lam]
        self.chol = np.linalg.cholesky(mats[-1].toarray())


def two_phase(ne, contrast, seed=0, fraction=0.4, radii=(1.0, 3.0)):
    """inclusion_field of the box ne with E_matrix = 1, E_inclusion = contrast."""
    from pcg_mpi_solver_b200.hexmesh import inclusion_field
    return inclusion_field(ne, fraction, radii, 1.0, float(contrast), seed)


def random_field(ne, seed, lo=0.1, hi=10.0):
    """Log-uniform per-element moduli in [lo, hi], shape (ne[2], ne[1], ne[0])."""
    rng = np.random.default_rng(seed)
    return np.exp(rng.uniform(np.log(lo), np.log(hi), (ne[2], ne[1], ne[0])))
