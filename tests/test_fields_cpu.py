"""The host restatement of the field recovery (tests/fields_cases.py, the arithmetic of csrc/fields.cuh) against physics,
independently of the GPU: a linear displacement gives its exact strain and stress in every element, the stress law carries
the element energy of hex_element_stiffness, principal values match eigvalsh and stay ordered on degenerate tensors, and
the node-level interface lists of a partition pair up."""
import numpy as np
import pytest

from pcg_mpi_solver_b200.hexmesh import HexBlock, block_grid, hex_element_stiffness, interface_node_lists, partition_blocks
from tests import fields_cases as C


def _linear_x(block, G):
    """Free-dof vector of u = G X, X the global node coordinates times h."""
    nx, ny, nz = block.ne
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(block.x_lo, nx + 1), indexing="ij")
    X = np.stack([lx.ravel() + block.e0[0], ly.ravel() + block.e0[1], lz.ravel() + block.e0[2]], axis=1) * block.h
    return (X @ G.T).ravel()


def _sym_voigt(G):
    e = 0.5 * (G + G.T)
    return np.array([e[0, 0], e[1, 1], e[2, 2], e[1, 2], e[0, 2], e[0, 1]])


def _sigma(eps, E, nu):
    lam, m2 = C.lam_m2(nu)
    tr = eps[:3].sum()
    return E * np.concatenate([lam * tr + m2 * eps[:3], m2 * eps[3:]])


@pytest.mark.parametrize("box,G_kind", [
    (((9, 7, 6), (2, 1, 3), (5, 4, 2)), "full"),     # away from the clamped face: any linear field
    (((6, 5, 4), (0, 0, 0), (6, 5, 4)), "x_only"),   # clamped line: u = G[:, 0] X vanishes at X = 0
])
def test_patch_linear_field(box, G_kind):
    ng, e0, ne = box
    blk = HexBlock(ng, e0, ne, h=0.37, E=2.5, nu=0.27)
    G = np.random.default_rng(3).standard_normal((3, 3))
    if G_kind == "x_only":
        G[:, 1:] = 0.0
    eps = C.strain(blk, _linear_x(blk, G))
    sig = C.stress(blk, eps)
    want_e = _sym_voigt(G)
    want_s = _sigma(want_e, blk.E, blk.nu)
    assert np.max(np.abs(eps - want_e[None, :])) <= 1e-14 * np.max(np.abs(want_e))
    assert np.max(np.abs(sig - want_s[None, :])) <= 1e-14 * np.max(np.abs(want_s))
    # a voxel field scales each element's stress by its own E
    f = np.random.default_rng(4).uniform(0.5, 20.0, tuple(reversed(ne)))
    sig_f = C.stress(blk, eps, f)
    assert np.max(np.abs(sig_f - f.reshape(-1, 1) * _sigma(want_e, 1.0, blk.nu)[None, :])) <= 1e-14 * np.max(np.abs(sig_f))


@pytest.mark.parametrize("nu,h,E", [(0.3, 1.0, 1.0), (0.2, 0.125, 7.0), (0.45, 0.37, 0.01)])
def test_energy_identity(nu, h, E):
    """Ck u^T Ke u = h^3 sigma : eps (Ck = E h) for a linear field on one element: the stress law is the operator's."""
    blk = HexBlock((3, 3, 3), (1, 1, 1), (1, 1, 1), h=h, E=E, nu=nu)
    for seed in range(5):
        G = np.random.default_rng(seed).standard_normal((3, 3))
        u = np.zeros(24)
        for l in range(8):
            X = (np.array([(l & 1) + 1, ((l >> 1) & 1) + 1, (l >> 2) + 1], dtype=float)) * h
            u[3 * l:3 * l + 3] = G @ X
        eps = C.strain(blk, _linear_x(blk, G))[0]
        sig = C.stress(blk, eps[None, :])[0]
        w = np.array([1, 1, 1, 2, 2, 2], dtype=float)
        lhs = E * h * (u @ hex_element_stiffness(1.0, nu) @ u)
        rhs = h ** 3 * np.sum(w * sig * eps)
        assert abs(lhs - rhs) <= 1e-14 * abs(rhs), (lhs, rhs)


def _voigt(M):
    return np.stack([M[:, 0, 0], M[:, 1, 1], M[:, 2, 2], M[:, 1, 2], M[:, 0, 2], M[:, 0, 1]], axis=1)


def test_principal_matches_eigvalsh():
    rng = np.random.default_rng(7)
    A = rng.standard_normal((20000, 3, 3)) * rng.uniform(1e-3, 1e3, (20000, 1, 1))
    M = 0.5 * (A + A.transpose(0, 2, 1))
    s = _voigt(M)
    keep = np.abs(C.bracket(s)) <= 0.99
    assert keep.sum() > 15000
    P = C.principal(s[keep])
    ev = np.sort(np.linalg.eigvalsh(M[keep]), axis=1)[:, ::-1]
    scale = np.max(np.abs(ev), axis=1, keepdims=True)
    assert np.max(np.abs(P - ev) / scale) <= 1e-12
    assert np.all(P[:, 0] >= P[:, 1]) and np.all(P[:, 1] >= P[:, 2])


def test_principal_special_tensors():
    a, b, t, p = 3.7, -1.25, 0.8, -2.5
    cases = {
        "zero": ([0, 0, 0, 0, 0, 0], [0, 0, 0]),
        "hydrostatic": ([p, p, p, 0, 0, 0], [p, p, p]),
        "uniaxial": ([a, 0, 0, 0, 0, 0], [a, 0, 0]),
        "uniaxial_neg": ([0, 0, b, 0, 0, 0], [0, 0, b]),
        "two_equal": ([a, b, b, 0, 0, 0], [a, b, b]),
        "pure_shear": ([0, 0, 0, 0, 0, t], [t, 0, -t]),
        "pure_shear_23": ([0, 0, 0, t, 0, 0], [t, 0, -t]),
    }
    for name, (s, want) in cases.items():
        P = C.principal(np.array([s], dtype=float))[0]
        assert np.all(np.isfinite(P)), name
        assert P[0] >= P[1] >= P[2], (name, P)
        assert np.max(np.abs(P - np.array(want, dtype=float))) <= 1e-7 * max(np.max(np.abs(s)), 1e-300), (name, P)
    # J2 pushed below zero by rounding (hydrostatic up to an ulp): I1 / 3 three times, no NaN
    s = np.array([[0.1, 0.1 + 2.0 ** -56, 0.1, 0, 0, 0]])
    P = C.principal(s)[0]
    assert np.all(np.isfinite(P)) and np.max(np.abs(P - 0.1)) <= 1e-15


def test_principal_order_on_degenerate_tensors():
    """P1 >= P2 >= P3 also where two or three values coincide and rounding alone separates them, and P2 is (I1 - P1) - P3
    wherever that lies between P3 and P1."""
    rng = np.random.default_rng(0)
    n = 20000
    Q = np.linalg.qr(rng.standard_normal((n, 3, 3)))[0]
    ev = rng.standard_normal((n, 3))
    ev[: n // 3, 1] = ev[: n // 3, 0]
    ev[n // 3: 2 * n // 3, 2] = ev[n // 3: 2 * n // 3, 1]
    ev[2 * n // 3:, :] = ev[2 * n // 3:, :1]
    s = _voigt(np.einsum("nij,nj,nkj->nik", Q, ev, Q))
    P = C.principal(s)
    assert np.all(np.isfinite(P))
    assert np.all(P[:, 0] >= P[:, 1]) and np.all(P[:, 1] >= P[:, 2])
    I1 = (s[:, 0] + s[:, 1]) + s[:, 2]
    p2 = (I1 - P[:, 0]) - P[:, 2]
    inside = (p2 <= P[:, 0]) & (p2 >= P[:, 2])
    assert np.array_equal(P[inside, 1], p2[inside])


def test_nodal_sums_count_incident_elements():
    blk = HexBlock((5, 4, 3), (0, 0, 0), (5, 4, 3))
    pv = np.random.default_rng(1).standard_normal((60, 3))
    S = C.nodal_sums(blk, pv)
    lz, ly, lx = np.meshgrid(np.arange(4), np.arange(5), np.arange(6), indexing="ij")
    inc = lambda l, n: np.where((l == 0) | (l == n), 1, 2)   # noqa: E731
    assert np.array_equal(S[:, 3], (inc(lx, 5) * inc(ly, 4) * inc(lz, 3)).ravel().astype(float))
    assert np.allclose(C.nodal_average(S)[0], pv[0])


@pytest.mark.parametrize("world", [2, 4, 8])
def test_interface_node_lists_pair_up(world):
    ng = (6, 5, 4)
    blocks = partition_blocks(ng, block_grid(world))

    def gid(b, local):
        nx1, ny1 = b.ne[0] + 1, b.ne[1] + 1
        lx, ly, lz = local % nx1, (local // nx1) % ny1, local // (nx1 * ny1)
        return ((lz + b.e0[2]) * (ng[1] + 1) + (ly + b.e0[1])) * (ng[0] + 1) + (lx + b.e0[0])

    lists = [dict(zip(*interface_node_lists(blocks, r))) for r in range(world)]
    saw_clamped = False
    for a in range(world):
        assert lists[a], a
        for b, la in lists[a].items():
            ga, gb = gid(blocks[a], la), gid(blocks[b], lists[b][a])
            assert np.array_equal(ga, gb) and np.all(np.diff(ga) > 0), (a, b)
            saw_clamped |= bool(np.any(ga % (ng[0] + 1) == 0))
            # exactly the nodes both boxes contain
            ra, rb = blocks[a].node_ranges(), blocks[b].node_ranges()
            gx, gy, gz = ga % (ng[0] + 1), (ga // (ng[0] + 1)) % (ng[1] + 1), ga // ((ng[0] + 1) * (ng[1] + 1))
            want = np.prod([min(ra[k][1], rb[k][1]) - max(ra[k][0], rb[k][0]) + 1 for k in range(3)])
            assert ga.size == want
            for k, g in enumerate((gx, gy, gz)):
                assert np.all(g >= max(ra[k][0], rb[k][0])) and np.all(g <= min(ra[k][1], rb[k][1]))
    assert saw_clamped == (world > 2)   # a cut across y shares nodes of the clamped line; a cut across x does not
