"""Host restatement of the multigrid preconditioner for boxes of any size (HexMultigrid(coarsening="any"),
pcgb_mg_create_any): the oracle of its tests.

Rule: every axis of a level is coarsened on its own while some axis has ne >= 3.  An axis with ne >= 3 is halved to
(ne + 1) / 2 elements, coarse node j at fine node s(j) = min(2j, ne) (an odd axis ends in a coarse element one fine element
wide at its high end); an axis with ne <= 2 is kept, s(j) = j.  Fine node i between s(j) and s(j+1) takes the weight
(s(j+1) - i) / (s(j+1) - s(j)) from coarse node j and the rest from j + 1, so P is the tensor product of three 1-D maps,
clamped x = 0 nodes dropped.  The coarse matrices are element-level Galerkin products with a coarse element of width w_a in
{1, 2} fine elements per axis and phi_0(p) = (w - p) / w, phi_1(p) = p / w; assembled, they equal scipy P^T A P.  The V-cycle
is gmg_cases.HostMultigrid's with these matrices and transfers.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import gmg_cases as G
from tests import voxel_cases as V

MAX_LEVELS = 32


def levels(ne, max_levels=MAX_LEVELS):
    """Element counts of every level; ValueError for a box with nothing to coarsen or more than max_levels levels."""
    out = [tuple(int(v) for v in ne)]
    while max(out[-1]) >= 3:
        out.append(tuple(v if v <= 2 else (v + 1) // 2 for v in out[-1]))
        if len(out) > max_levels:
            raise ValueError("more than %d levels" % max_levels)
    if len(out) < 2:
        raise ValueError("nothing to coarsen")
    return out


def positions(nf):
    """s(j), j = 0 .. nc: the fine node of every coarse node of an axis of nf fine elements."""
    if nf <= 2:
        return np.arange(nf + 1)
    nc = (nf + 1) // 2
    return np.minimum(2 * np.arange(nc + 1), nf)


def interp_1d(s):
    """(nf + 1) x (nc + 1) dense 1-D interpolation from the coarse positions s (fine node s[-1] is the last)."""
    nf = int(s[-1])
    P = np.zeros((nf + 1, len(s)))
    for j in range(len(s) - 1):
        a, b = int(s[j]), int(s[j + 1])
        for i in range(a, b):
            P[i, j] = (b - i) / (b - a)
            P[i, j + 1] = (i - a) / (b - a)
    P[nf, len(s) - 1] = 1.0
    return P


def prolongation_any(ne_f, pos=positions):
    """P (free dofs of level ne_f x free dofs of its coarse level), scipy CSR: the tensor product of the 1-D maps, clamped
    nodes dropped.  pos: the position rule of an axis (a variant's can be tested against it)."""
    Px, Py, Pz = (sp.csr_matrix(interp_1d(pos(ne_f[a]))) for a in range(3))
    Pn = sp.kron(Pz, sp.kron(Py, Px)).tocsr()
    nfx, ncx = ne_f[0] + 1, Px.shape[1]
    keep_f = np.arange(Pn.shape[0]) % nfx >= 1
    keep_c = np.arange(Pn.shape[1]) % ncx >= 1
    Pn = Pn[keep_f][:, keep_c]
    return sp.kron(Pn, sp.identity(3)).tocsr()


def child_weight(c, l, k, thin):
    """Weight of coarse corner k on child c's node l: prod_a phi_{k_a}(p_a), p = c_a + bit_a(l), w_a = 1 where bit a of thin."""
    w = 1.0
    for a in range(3):
        p = ((c >> a) & 1) + ((l >> a) & 1)
        wa = 1 if (thin >> a) & 1 else 2
        w *= p / wa if (k >> a) & 1 else (wa - p) / wa
    return w


def child_Q(c, thin):
    Q = np.zeros((24, 24))
    for l in range(8):
        for k in range(8):
            for d in range(3):
                Q[3 * l + d, 3 * k + d] = child_weight(c, l, k, thin)
    return Q


def _axis_groups(nf):
    """Groups of coarse elements of one axis with equal width: (coarse slice, width, fine start for child c_a)."""
    if nf <= 2:
        return [(slice(0, nf), 1, lambda c: slice(0, nf))]
    full = nf // 2
    g = [(slice(0, full), 2, lambda c, full=full: slice(c, c + 2 * full, 2))]
    if nf % 2:
        g.append((slice(full, full + 1), 1, lambda c, nf=nf: slice(nf - 1, nf)))
    return g


def galerkin_any(kf):
    """Coarse element matrices of fine ones kf (nz, ny, nx, 24, 24) under the rule: K_E = sum_c Q_c^T K_child(c) Q_c over the
    children that exist."""
    nz, ny, nx = kf.shape[:3]
    nc = [len(positions(n)) - 1 for n in (nx, ny, nz)]
    out = np.zeros((nc[2], nc[1], nc[0], 24, 24))
    for sz, wz, fz in _axis_groups(nz):
        for sy, wy, fy in _axis_groups(ny):
            for sx, wx, fx in _axis_groups(nx):
                thin = (wx == 1) | ((wy == 1) << 1) | ((wz == 1) << 2)
                for c in range(8):
                    cx, cy, cz = c & 1, (c >> 1) & 1, c >> 2
                    if cx >= wx or cy >= wy or cz >= wz:
                        continue
                    Q = child_Q(c, thin)
                    out[sz, sy, sx] += Q.T @ kf[fz(cz), fy(cy), fx(cx)] @ Q
    return out


def level_elements(field, h, nu=0.3):
    """Element matrices of every level: [fine, Galerkin level 1, ...]."""
    ne = tuple(int(v) for v in reversed(field.shape))
    out = [V.fine_elements(field, h, R.hex_ke(1.0, nu))]
    for _ in levels(ne)[1:]:
        out.append(galerkin_any(out[-1]))
    return out


def level_matrices(field, h, nu=0.3):
    return [V.assemble(k, None) for k in level_elements(field, h, nu)]


def ptap_matrices(field, h, nu=0.3):
    """Every level as scipy P^T A P from the fine voxel matrix."""
    lv = levels(tuple(int(v) for v in reversed(field.shape)))
    mats = [V.field_csr(field, h, nu)]
    for l in range(len(lv) - 1):
        P = prolongation_any(lv[l])
        mats.append((P.T @ mats[-1] @ P).tocsr())
    return mats


class HostAnyMultigrid(G.HostMultigrid):
    """HostMultigrid's V-cycle on the levels of the any rule.  lambdas / minv: as in HostMultigrid; mats: level matrices."""

    def __init__(self, field, h, degree=2, lo=0.25, lambdas=None, minv=None, nu=0.3, mats=None):
        ne = tuple(int(v) for v in reversed(field.shape))
        self.ne = levels(ne)
        self.degree, self.lo = degree, lo
        self.mats = level_matrices(field, h, nu) if mats is None else mats
        self.A = [V.MatOp(A) for A in self.mats]
        self.P = [prolongation_any(n_) for n_ in self.ne[:-1]]
        self.dinv = [1.0 / A.diag for A in self.A]
        if minv is not None:
            self.dinv[0] = minv
        L = len(self.ne)
        self.lam = list(lambdas[:L - 1]) if lambdas is not None else [G.lanczos_lambda(self.A[l], self.dinv[l]) for l in range(L - 1)]
        self.coef = [G.cheb_coeffs(lam, degree, lo) for lam in self.lam]
        self.chol = np.linalg.cholesky(self.mats[-1].toarray())

    def apply(self, r):
        L = len(self.ne)
        b, x = [None] * L, [None] * L
        b[0] = r
        for l in range(L - 1):
            x[l], res = self.smooth(l, b[l], None, True, resid=True)
            b[l + 1] = self.P[l].T @ res
        x[L - 1] = self.coarse_solve(b[L - 1])
        for l in range(L - 2, -1, -1):
            x[l] = x[l] + self.P[l] @ x[l + 1]
            x[l], _ = self.smooth(l, b[l], x[l], False)
        return x[0]


def uniform_field(ne, E=1.0):
    """The field of a uniform box of modulus E: what pcgb_mg_create_any builds without one (Ck = E h per element)."""
    return np.full((ne[2], ne[1], ne[0]), float(E))


# boxes whose Galerkin coarsest matrix at gmg_cases.BAD_NU has a negative eigenvalue (pinned in test_gmg_galerkin_cpu.py):
# the field path on a random field of BAD_NU_FIELD_BOX, the any rule on BAD_NU_ANY_BOX uniform and with a random field;
# the fields are voxel_cases.random_field(box, seed=sum(box))
BAD_NU_FIELD_BOX, BAD_NU_ANY_BOX = (8, 8, 8), (9, 7, 5)


def field_of(ne, contrast, seed=0):
    """The test field of a box: uniform 1 at contrast 1, else V.two_phase (inclusions of modulus `contrast`)."""
    if contrast == 1:
        return np.ones((ne[2], ne[1], ne[0]))
    return V.two_phase(ne, contrast, seed=seed)


def host_pcg_iters(ne, contrast, tol=1e-8, degree=2, seed=0):
    """Host MG-PCG iterations on box ne (h = 1 / ne[0]) with the load of hexmesh.load_vector."""
    f = field_of(ne, contrast, seed)
    h = 1.0 / ne[0]
    H = HostAnyMultigrid(f, h, degree=degree)
    b = G.load_vector(ne, h)
    _, it = G.pcg(H.mats[0], b, H.apply, tol, 500)
    return it


# box -> levels under the any rule (the tables of DESIGN §2.6)
LEVELS = {
    (16, 16, 16): [(16, 16, 16), (8, 8, 8), (4, 4, 4), (2, 2, 2)],
    (24, 24, 24): [(24, 24, 24), (12, 12, 12), (6, 6, 6), (3, 3, 3), (2, 2, 2)],
    (16, 16, 15): [(16, 16, 15), (8, 8, 8), (4, 4, 4), (2, 2, 2)],
    (15, 15, 15): [(15, 15, 15), (8, 8, 8), (4, 4, 4), (2, 2, 2)],
    (17, 17, 17): [(17, 17, 17), (9, 9, 9), (5, 5, 5), (3, 3, 3), (2, 2, 2)],
    (25, 25, 25): [(25, 25, 25), (13, 13, 13), (7, 7, 7), (4, 4, 4), (2, 2, 2)],
    (25, 17, 9): [(25, 17, 9), (13, 9, 5), (7, 5, 3), (4, 3, 2), (2, 2, 2)],
    (38, 4, 16): [(38, 4, 16), (19, 2, 8), (10, 2, 4), (5, 2, 2), (3, 2, 2), (2, 2, 2)],
    (1, 5, 9): [(1, 5, 9), (1, 3, 5), (1, 2, 3), (1, 2, 2)],
    (3, 3, 3): [(3, 3, 3), (2, 2, 2)],
}
