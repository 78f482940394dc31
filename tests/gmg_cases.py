"""Host restatement of the geometric multigrid preconditioner (pcgb_mg_*, csrc/gmg.cuh): the oracle of its tests.

Same hierarchy, coefficients and order of operations as the library: nested hex boxes (every ne halved while all are even
and the halves stay >= 2), trilinear P on the free nodes (x fastest, global x = 0 clamped, dof = 3 node + dir), Chebyshev
smoothing of D^-1 A on [lo, 1.1] * lambda with lambda from 20 Lanczos steps, a dense solve on the coarsest box.  Operators are
applied matrix-free with numpy (the Q1 element of oracle/ref_pcg.hex_ke), which keeps 64^3 affordable on a CPU.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import ref_pcg as R

LANCZOS_STEPS = 20


def levels_of(ne):
    out = [tuple(int(v) for v in ne)]
    while all(v % 2 == 0 and v // 2 >= 2 for v in out[-1]):
        out.append(tuple(v // 2 for v in out[-1]))
    return out


def nfree(ne):
    return ne[0] * (ne[1] + 1) * (ne[2] + 1)


def start_vector(n):
    i = np.arange(n, dtype=np.int64)
    return 0.5 + ((37 * i + 11) % 101).astype(np.float64) / 101.0


class HexOp:
    """y = A x of the clamped box ne (spacing h, Young's modulus E, Poisson ratio nu) in the free-dof numbering, matrix-free.
    The element matrix is that of R.hex_box_csr: hex_ke(1, nu) * (E h)."""

    def __init__(self, ne, h, nu=0.3, E=1.0):
        self.ne = tuple(ne)
        self.ke = R.hex_ke(1.0, nu) * (E * h)
        self.n = 3 * nfree(ne)
        nx, ny, nz = ne
        d = np.zeros((nz + 1, ny + 1, nx + 1, 3))
        kd = np.diag(self.ke)
        for l in range(8):
            ox, oy, oz = l & 1, (l >> 1) & 1, (l >> 2) & 1
            d[oz:oz + nz, oy:oy + ny, ox:ox + nx] += kd[3 * l:3 * l + 3]
        self.diag = d[:, :, 1:].reshape(-1).copy()

    def full(self, v):
        nx, ny, nz = self.ne
        u = np.zeros((nz + 1, ny + 1, nx + 1, 3), dtype=v.dtype)
        u[:, :, 1:] = v.reshape(nz + 1, ny + 1, nx, 3)
        return u

    def __matmul__(self, v):
        nx, ny, nz = self.ne
        u = self.full(v)
        X = np.concatenate([u[(l >> 2) & 1:((l >> 2) & 1) + nz, (l >> 1) & 1:((l >> 1) & 1) + ny, l & 1:(l & 1) + nx]
                            for l in range(8)], axis=3)
        Y = X @ self.ke.T
        y = np.zeros_like(u)
        for l in range(8):
            ox, oy, oz = l & 1, (l >> 1) & 1, (l >> 2) & 1
            y[oz:oz + nz, oy:oy + ny, ox:ox + nx] += Y[..., 3 * l:3 * l + 3]
        return y[:, :, 1:].reshape(-1)


def prolongation_matrix(ne_f):
    """P (n_f x n_c, scipy CSR): trilinear interpolation of the coarse free nodes (box ne_f / 2) onto the fine ones."""
    ne_c = tuple(v // 2 for v in ne_f)
    rows, cols, vals = [], [], []
    fz, fy, fx = np.meshgrid(np.arange(ne_f[2] + 1), np.arange(ne_f[1] + 1), np.arange(1, ne_f[0] + 1), indexing="ij")
    fz, fy, fx = fz.ravel(), fy.ravel(), fx.ravel()
    fnode = np.arange(fx.size)
    for kz in (0, 1):
        for ky in (0, 1):
            for kx in (0, 1):
                cz, cy, cx = (fz >> 1) + kz, (fy >> 1) + ky, (fx >> 1) + kx
                w = np.ones(fx.size)
                for f, k in ((fz, kz), (fy, ky), (fx, kx)):
                    w *= np.where(f % 2 == 1, 0.5, np.where(k == 0, 1.0, 0.0))
                ok = (w > 0) & (cx >= 1)
                cnode = (cz * (ne_c[1] + 1) + cy) * ne_c[0] + (cx - 1)
                for d in range(3):
                    rows.append(3 * fnode[ok] + d)
                    cols.append(3 * cnode[ok] + d)
                    vals.append(w[ok])
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                         shape=(3 * nfree(ne_f), 3 * nfree(ne_c)))


def _grid(v, ne):
    nx, ny, nz = ne
    u = np.zeros((nz + 1, ny + 1, nx + 1, 3), dtype=v.dtype)
    u[:, :, 1:] = v.reshape(nz + 1, ny + 1, nx, 3)
    return u


def restrict(rf, ne_f, dtype=np.float64):
    """r_c = P^T r_f as the kernel gathers it: per coarse node, fine offsets (dz, dy, dx) ascending, from 0.  Also returns
    the sum of |terms| per entry (for rounding bounds)."""
    ne_c = tuple(v // 2 for v in ne_f)
    u = np.pad(_grid(rf.astype(dtype), ne_f), ((1, 1), (1, 1), (1, 1), (0, 0)))
    s = np.zeros((ne_c[2] + 1, ne_c[1] + 1, ne_c[0] + 1, 3), dtype=dtype)
    a = np.zeros_like(s)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                w = dtype((0.5 if dx else 1.0) * (0.5 if dy else 1.0) * (0.5 if dz else 1.0))
                t = w * u[1 + dz: 1 + dz + 2 * ne_c[2] + 1: 2, 1 + dy: 1 + dy + 2 * ne_c[1] + 1: 2, 1 + dx: 1 + dx + 2 * ne_c[0] + 1: 2]
                s = s + t
                a = a + np.abs(t)
    return s[:, :, 1:].reshape(-1), a[:, :, 1:].reshape(-1)


def prolong_add(ec, xf, ne_f, dtype=np.float64):
    """x_f + P e_c as the kernel gathers it: per fine node, coarse nodes (z, y, x) ascending, summed from 0, then added."""
    ne_c = tuple(v // 2 for v in ne_f)
    u = np.pad(_grid(ec.astype(dtype), ne_c), ((0, 1), (0, 1), (0, 1), (0, 0)))
    f = [np.arange(ne_f[a] + 1) for a in range(3)]
    s = np.zeros((ne_f[2] + 1, ne_f[1] + 1, ne_f[0] + 1, 3), dtype=dtype)
    a = np.zeros_like(s)
    for kz in (0, 1):
        for ky in (0, 1):
            for kx in (0, 1):
                ws = [np.where(f[ax] % 2 == 1, 0.5, 1.0 if k == 0 else 0.0) for ax, k in ((0, kx), (1, ky), (2, kz))]
                w = (ws[2][:, None, None] * ws[1][None, :, None] * ws[0][None, None, :]).astype(dtype)
                t = w[..., None] * u[(f[2] >> 1) + kz][:, (f[1] >> 1) + ky][:, :, (f[0] >> 1) + kx]
                s = s + t
                a = a + np.abs(t)
    s, a = s[:, :, 1:].reshape(-1), a[:, :, 1:].reshape(-1)
    return xf.astype(dtype) + s, np.abs(xf).astype(dtype) + a


def cheb_coeffs(lam, degree, lo):
    a, b = lo * lam, 1.1 * lam
    theta, delta = 0.5 * (b + a), 0.5 * (b - a)
    sigma = theta / delta
    rho = 1.0 / sigma
    c1, c2 = [], []
    for _ in range(1, degree):
        rn = 1.0 / (2.0 * sigma - rho)
        c1.append(rn * rho)
        c2.append(2.0 * rn / delta)
        rho = rn
    return 1.0 / theta, c1, c2


def lanczos_lambda(A, dinv, steps=LANCZOS_STEPS):
    """Largest eigenvalue of D^-1 A: Lanczos in the D inner product from start_vector, then the tridiagonal's top eigenvalue."""
    v = start_vector(A.n)
    v = v * (1.0 / np.sqrt(np.dot(v, v / dinv)))
    vp, beta, al, be = np.zeros_like(v), 0.0, [], []
    for it in range(steps):
        y = A @ v
        al.append(np.dot(v, y))
        if it + 1 == steps:
            break
        w = dinv * y - al[-1] * v - beta * vp
        beta = np.sqrt(np.dot(w, w / dinv))
        be.append(beta)
        vp, v = v, w * (1.0 / beta)
    return np.linalg.eigvalsh(np.diag(al) + np.diag(be, 1) + np.diag(be, -1))[-1]


class HostMultigrid:
    """The V-cycle of pcgb_mg_apply on the host.  lambdas: use these estimates (e.g. the device's) instead of computing them.
    E, nu: the material of every level (the coarse matrices are rediscretised with the fine level's E and nu)."""

    def __init__(self, ne, h, degree=2, lo=0.25, lambdas=None, minv=None, E=1.0, nu=0.3):
        self.ne = levels_of(ne)
        self.degree, self.lo = degree, lo
        self.A = [HexOp(n_, h * 2 ** l, nu=nu, E=E) for l, n_ in enumerate(self.ne)]
        self.dinv = [1.0 / A.diag for A in self.A]
        if minv is not None:
            self.dinv[0] = minv
        L = len(self.ne)
        self.lam = list(lambdas[:L - 1]) if lambdas is not None else [lanczos_lambda(self.A[l], self.dinv[l]) for l in range(L - 1)]
        self.coef = [cheb_coeffs(lam, degree, lo) for lam in self.lam]
        nec = self.ne[-1]
        Ac = R.hex_box_csr(nec, (0, 0, 0), nec, E=E, nu=nu, h=h * 2 ** (L - 1)).toarray()
        self.chol = np.linalg.cholesky(Ac)

    def coarse_solve(self, r):
        import scipy.linalg as sl
        y = sl.solve_triangular(self.chol, r, lower=True)
        return sl.solve_triangular(self.chol.T, y, lower=False)

    def smooth(self, l, b, x, zero_start, resid=False):
        A, dinv = self.A[l], self.dinv[l]
        inv_theta, c1, c2 = self.coef[l]
        r = b.copy() if zero_start else b - A @ x
        d = inv_theta * (dinv * r)
        x = d.copy() if zero_start else x + d
        for j in range(len(c1)):
            r = r - A @ d
            d = c1[j] * d + c2[j] * (dinv * r)
            x = x + d
        if resid:
            r = r - A @ d
        return x, r

    def apply(self, r):
        L = len(self.ne)
        b, x = [None] * L, [None] * L
        b[0] = r
        for l in range(L - 1):
            x[l], res = self.smooth(l, b[l], None, True, resid=True)
            b[l + 1] = restrict(res, self.ne[l])[0]
        x[L - 1] = self.coarse_solve(b[L - 1])
        for l in range(L - 2, -1, -1):
            x[l] = prolong_add(x[l + 1], x[l], self.ne[l])[0]
            x[l], _ = self.smooth(l, b[l], x[l], False)
        return x[0]


# fine box -> dofs of its coarsest level: both sides of one 1024-thread pass of the one-CTA Cholesky kernels (1020 | 1026,
# and n - k - 1 = 1024 inside 1026 and 1029), the smallest level and the largest one allowed
COARSE_SIZES = {(4, 4, 4): 54, (6, 6, 6): 144, (14, 14, 10): 1008, (10, 6, 32): 1020, (4, 16, 36): 1026, (14, 12, 12): 1029,
                (16, 14, 14): 1536}
# materials and spacings of the material tests: (E, nu, h)
MATERIALS = [(E, nu, h) for E in (7.5, 210.0) for nu in (0.2, 0.45) for h in (0.125, 2.0)]
# a Poisson ratio above 1/2: negative bulk modulus, indefinite stiffness matrices
BAD_NU_BOX, BAD_NU = (8, 8, 8), 0.6


def coarsest_matrix(ne, h, E=1.0, nu=0.3):
    """Dense matrix of the coarsest level of the fine box ne (spacing h), as pcgb_mg_create factors it."""
    lv = levels_of(ne)
    return R.hex_box_csr(lv[-1], (0, 0, 0), lv[-1], E=E, nu=nu, h=h * 2 ** (len(lv) - 1)).toarray()


def refined_solve(A, r):
    """A^-1 r by numpy, refined once with the residual r - A z summed in long double: the reference of the coarse solve."""
    z = np.linalg.solve(A, r)
    res = r.astype(np.longdouble) - A.astype(np.longdouble) @ z.astype(np.longdouble)
    return z + np.linalg.solve(A, res.astype(np.float64))


def pcg(A, b, M, tol, maxiter):
    """Plain PCG from x = 0; returns (x, iterations to ||r|| <= tol ||b||)."""
    x = np.zeros_like(b)
    r = b.copy()
    tolb = tol * np.linalg.norm(b)
    rho_prev, p = None, None
    for i in range(maxiter):
        z = M(r)
        rho = np.dot(z, r)
        p = z if p is None else z + (rho / rho_prev) * p
        q = A @ p
        alpha = rho / np.dot(p, q)
        x = x + alpha * p
        r = r - alpha * q
        rho_prev = rho
        if np.linalg.norm(r) <= tolb:
            return x, i + 1
    return x, maxiter


def load_vector(ne, h):
    """b of hexmesh.load_vector for the whole box (traction -z on x = max)."""
    nx, ny, nz = ne
    b = np.zeros((nz + 1, ny + 1, nx, 3))
    cy = np.where((np.arange(ny + 1) == 0) | (np.arange(ny + 1) == ny), 0.5, 1.0)
    cz = np.where((np.arange(nz + 1) == 0) | (np.arange(nz + 1) == nz), 0.5, 1.0)
    b[:, :, nx - 1, 2] = -h * h * cz[:, None] * cy[None, :]
    return b.reshape(-1)
