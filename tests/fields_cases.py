"""Host restatement of the field recovery of csrc/fields.cuh (HexFields): the same operations, in the same order, elementwise in
numpy (which rounds every operation and never contracts), so element strain and stress are bit-identical to the kernels;
principal values use numpy's arccos / cos, so they agree to the accuracy of arccos near +-1.  Shared by the CPU tests
(against physics: patch test, energy identity, eigvalsh) and the GPU tests (against the kernels)."""
from __future__ import annotations

import numpy as np

A1 = 1.0 / 3.0


def lam_m2(nu: float):
    """lambda and 2 mu of hexmesh.hex_element_stiffness(1.0, nu), as that function computes them."""
    E = 1.0
    lam = E * nu / ((1 + nu) * (1 - 2 * nu))
    mu = E / (2 * (1 + nu))
    return lam, 2 * mu


def all_nodes_u(block, x: np.ndarray) -> np.ndarray:
    """(nodes, 3) displacement of every node of the box (node = (lz (ny+1) + ly) (nx+1) + lx), 0.0 on the clamped line."""
    nx, ny, nz = block.ne
    U = np.zeros(((nz + 1) * (ny + 1) * (nx + 1), 3))
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    free = np.nonzero(lx.ravel() >= block.x_lo)[0]
    U[free] = np.asarray(x, dtype=np.float64).reshape(-1, 3)
    return U


def element_nodes(block) -> np.ndarray:
    """(8, ne) node of local node la of each element: the reference's ElemList_LocNodeIdVector layout."""
    nx, ny, nz = block.ne
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex, ey, ez = ex.ravel(), ey.ravel(), ez.ravel()
    return np.stack([((ez + (l >> 2)) * (ny + 1) + (ey + ((l >> 1) & 1))) * (nx + 1) + (ex + (l & 1)) for l in range(8)])


def strain(block, x: np.ndarray) -> np.ndarray:
    """(ne, 6) element strain, Voigt (11, 22, 33, 23, 13, 12), tensor shears: the centroid Q1 gradient."""
    U = all_nodes_u(block, x)
    Ue = U[element_nodes(block)]                      # (8, ne, 3)
    q = 0.25 / block.h
    g = np.empty((3, 3, Ue.shape[1]))
    for a in range(3):
        for i in range(3):
            acc = np.zeros(Ue.shape[1])
            for l in range(8):
                acc = acc + Ue[l, :, i] if (l >> a) & 1 else acc - Ue[l, :, i]
            g[a, i] = acc * q
    eps = np.empty((Ue.shape[1], 6))
    eps[:, 0], eps[:, 1], eps[:, 2] = g[0, 0], g[1, 1], g[2, 2]
    eps[:, 3] = 0.5 * (g[1, 2] + g[2, 1])
    eps[:, 4] = 0.5 * (g[0, 2] + g[2, 0])
    eps[:, 5] = 0.5 * (g[0, 1] + g[1, 0])
    return eps


def stress(block, eps: np.ndarray, E_field=None) -> np.ndarray:
    """(ne, 6) sigma = E_e D eps."""
    lam, m2 = lam_m2(block.nu)
    E = np.full(eps.shape[0], float(block.E)) if E_field is None else np.asarray(E_field, dtype=np.float64).reshape(-1)
    tr = (eps[:, 0] + eps[:, 1]) + eps[:, 2]
    ltr = lam * tr
    s = np.empty_like(eps)
    for k in range(3):
        s[:, k] = E * (ltr + m2 * eps[:, k])
    for k in range(3, 6):
        s[:, k] = E * (m2 * eps[:, k])
    return s


def invariants(s: np.ndarray):
    s11, s22, s33, s23, s13, s12 = (s[:, k] for k in range(6))
    s12_2, s23_2, s13_2 = s12 * s12, s23 * s23, s13 * s13
    I1 = (s11 + s22) + s33
    I2 = s11 * s22 + s22 * s33 + s33 * s11 - s12_2 - s23_2 - s13_2
    I3 = s11 * s22 * s33 - s11 * s23_2 - s22 * s13_2 - s33 * s12_2 + 2.0 * s12 * s23 * s13
    return I1, I2, I3


def bracket(s: np.ndarray) -> np.ndarray:
    """0.5 (2 I1^3 - 9 I1 I2 + 27 I3) / J2^1.5, unclamped (nan where J2 <= 0)."""
    I1, I2, I3 = invariants(s)
    J2 = I1 * I1 - 3.0 * I2
    with np.errstate(divide="ignore", invalid="ignore"):
        return 0.5 * (2.0 * (I1 * I1 * I1) - 9.0 * I1 * I2 + 27.0 * I3) / (J2 * np.sqrt(np.maximum(J2, 0.0)))


def principal(s: np.ndarray) -> np.ndarray:
    """(N, 3) P1 >= P2 >= P3 of the symmetric tensors s (N, 6): getPrincipalStress without the 1e-24 max|S| term, I1 / 3
    where J2 sqrt(J2) <= 0, and P2 = (I1 - P1) - P3 clamped to [P3, P1]."""
    I1, I2, I3 = invariants(s)
    I1_2 = I1 * I1
    I1_3 = I1_2 * I1
    J2 = I1_2 - 3.0 * I2
    rj = np.sqrt(np.maximum(J2, 0.0))
    den = J2 * rj
    ok = den > 0.0
    c = A1 * I1
    P = np.repeat(c[None, :], 3, axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        br = (0.5 * ((2.0 * I1_3 - 9.0 * I1 * I2) + 27.0 * I3)) / den
    br = np.clip(np.where(ok, br, 0.0), -1.0, 1.0)
    phi = A1 * np.arccos(br)
    f = (2.0 * A1) * rj
    P[0] = np.where(ok, c + f * np.cos(phi), c)
    P[1] = np.where(ok, c + f * np.cos(phi + (2.0 * A1) * np.pi), c)
    P[2] = np.where(ok, c + f * np.cos(phi + (4.0 * A1) * np.pi), c)
    hi, lo = P.max(axis=0), P.min(axis=0)
    return np.stack([hi, np.minimum(np.maximum((I1 - hi) - lo, lo), hi), lo], axis=1)


def nodal_sums(block, pv: np.ndarray) -> np.ndarray:
    """(nodes, 4) (sum_0, sum_1, sum_2, count) of the element values pv (ne, 3): np.bincount over the (8, ne) node array
    ravelled (ascending la, then ascending element), as getNodalPS sums them (pcg_solver.py:764-771)."""
    nodes = element_nodes(block).ravel()
    nn = int(np.prod([v + 1 for v in block.ne]))
    out = np.empty((nn, 4))
    for i in range(3):
        w = (pv[:, i] * np.ones(8)[:, None]).ravel()
        out[:, i] = np.bincount(nodes, weights=w, minlength=nn)
    out[:, 3] = np.bincount(nodes, weights=np.ones(nodes.size), minlength=nn)
    return out


def nodal_average(sums: np.ndarray) -> np.ndarray:
    return sums[:, :3] / (sums[:, 3:4] + 1e-15)


def smooth_x(block) -> np.ndarray:
    """A deterministic smooth displacement of the box's free dofs from its GLOBAL node coordinates (so the boxes of a
    partition see the global mesh's values)."""
    nx, ny, nz = block.ne
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(block.x_lo, nx + 1), indexing="ij")
    X = (lx.ravel() + block.e0[0]) / block.ng[0]
    Y = (ly.ravel() + block.e0[1]) / block.ng[1]
    Z = (lz.ravel() + block.e0[2]) / block.ng[2]
    u = np.stack([np.sin(1.3 * X + 0.7 * Y) * (1.0 + Z), 0.4 * X * X - np.cos(2.1 * Z + Y), X * Y * Z + 0.25 * np.sin(3.0 * Y)], axis=1)
    return np.ascontiguousarray(u.ravel() * 1e-3)


def restrict_x(global_block, gx: np.ndarray, block) -> np.ndarray:
    """The entries of the global mesh's free-dof vector gx (global_block: the whole mesh as one box) at the free nodes of
    `block`, in the box's free numbering."""
    ng = global_block.ng
    nx, ny, nz = block.ne
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(block.x_lo, nx + 1), indexing="ij")
    g = ((lz.ravel() + block.e0[2]) * (ng[1] + 1) + (ly.ravel() + block.e0[1])) * ng[0] + (lx.ravel() + block.e0[0] - 1)
    return np.ascontiguousarray(gx.reshape(-1, 3)[g].ravel())


def global_elements(block) -> np.ndarray:
    """Global element ids (x fastest over the mesh) of the box's elements, in the box's element order."""
    ng = block.ng
    z, y, x = np.meshgrid(*[np.arange(block.e0[a], block.e0[a] + block.ne[a]) for a in (2, 1, 0)], indexing="ij")
    return ((z * ng[1] + y) * ng[0] + x).ravel()


def global_nodes(block) -> np.ndarray:
    """Global node ids (clamped line included) of every node of the box, in the box's node order."""
    ng = block.ng
    z, y, x = np.meshgrid(*[np.arange(block.e0[a], block.e0[a] + block.ne[a] + 1) for a in (2, 1, 0)], indexing="ij")
    return ((z * (ng[1] + 1) + y) * (ng[0] + 1) + x).ravel()
