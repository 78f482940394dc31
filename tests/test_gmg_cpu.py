"""CPU checks of the geometric multigrid preconditioner: the transfer operator against the rediscretised coarse matrices,
the host V-cycle (the oracle of tests/test_gpu_gmg.py) against its iteration-count target, and the C ABI without a GPU."""
import ctypes

import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import gmg_cases as G


@pytest.mark.parametrize("ne", [(2, 4, 8), (16, 8, 4), (4, 4, 4), (6, 2, 4)])
def test_galerkin_product_equals_rediscretised_coarse_matrix(ne):
    h = 0.125
    Af = R.hex_box_csr(ne, (0, 0, 0), ne, h=h)
    nec = tuple(v // 2 for v in ne)
    Ac = R.hex_box_csr(nec, (0, 0, 0), nec, h=2 * h).toarray()
    P = G.prolongation_matrix(ne)
    Gc = (P.T @ Af @ P).toarray()
    scale = np.abs(Ac).max()
    assert np.abs(Gc - Ac).max() <= 1e-13 * scale


@pytest.mark.parametrize("ne", [(2, 4, 8), (8, 6, 4)])
def test_gather_transfers_equal_the_matrix(ne):
    rng = np.random.default_rng(1)
    P = G.prolongation_matrix(ne)
    rf = rng.standard_normal(P.shape[0])
    ec = rng.standard_normal(P.shape[1])
    xf = rng.standard_normal(P.shape[0])
    assert np.allclose(G.restrict(rf, ne)[0], P.T @ rf, rtol=0, atol=1e-13 * np.abs(rf).sum())
    assert np.allclose(G.prolong_add(ec, xf, ne)[0], xf + P @ ec, rtol=0, atol=1e-13 * np.abs(ec).sum())


def test_levels_follow_the_coarsening_rule():
    assert G.levels_of((128, 128, 128))[-1] == (2, 2, 2) and len(G.levels_of((128, 128, 128))) == 7
    assert 3 * G.nfree((2, 2, 2)) == 54
    assert G.levels_of((16, 14, 14)) == [(16, 14, 14), (8, 7, 7)] and 3 * G.nfree((8, 7, 7)) == 1536
    assert len(G.levels_of((16, 16, 15))) == 1 and len(G.levels_of((2, 4, 8))) == 1


def test_lanczos_estimate_matches_eigsh():
    import scipy.sparse as sp
    import scipy.sparse.linalg as sla
    m = 8
    A = R.hex_box_csr((m, m, m), (0, 0, 0), (m, m, m), h=1.0 / m)
    s = sp.diags(1.0 / np.sqrt(A.diagonal()))
    top = sla.eigsh(s @ A @ s, k=1, which="LA", return_eigenvectors=False)[0]
    op = G.HexOp((m, m, m), 1.0 / m)
    assert abs(G.lanczos_lambda(op, 1.0 / op.diag) - top) <= 1e-3 * top


MATERIAL_BOXES = [(16, 8, 8), (8, 8, 8), (32, 16, 8), (24, 12, 12)]


@pytest.mark.parametrize("ne", MATERIAL_BOXES)
@pytest.mark.parametrize("E,nu,h", G.MATERIALS)
def test_host_operator_with_material_equals_the_assembled_matrix(ne, E, nu, h):
    """HexOp(E, nu, h) is R.hex_box_csr(E=, nu=, h=) on every level of the boxes the material tests use, and
    HostMultigrid passes its material to every level."""
    rng = np.random.default_rng(len(ne) + int(E))
    H = G.HostMultigrid(ne, h, E=E, nu=nu, lambdas=[1.0] * 8)
    for l, nel in enumerate(G.levels_of(ne)):
        A = R.hex_box_csr(nel, (0, 0, 0), nel, E=E, nu=nu, h=h * 2 ** l)
        v = rng.standard_normal(A.shape[0])
        ref = A @ v
        assert np.abs(H.A[l] @ v - ref).max() <= 1e-13 * np.abs(ref).max(), (l, nel)
        assert np.abs(H.A[l].diag - A.diagonal()).max() <= 1e-14 * A.diagonal().max(), (l, nel)
    Ac = G.coarsest_matrix(ne, h, E, nu)
    assert np.abs(H.chol @ H.chol.T - Ac).max() <= 1e-13 * np.abs(Ac).max()


def test_material_defaults_leave_the_host_operator_bit_identical():
    a, b = G.HexOp((8, 4, 4), 0.125), G.HexOp((8, 4, 4), 0.125, nu=0.3, E=1.0)
    assert np.array_equal(a.ke, R.hex_ke(1.0, 0.3) * 0.125) and np.array_equal(a.ke, b.ke)


# (box, E, nu, h, relative bound).  20 Lanczos steps resolve the top of the spectrum to 1e-5 or better at nu = 0.45 and at
# 16^3 with nu = 0.3, but the clustered top at nu = 0.2 leaves 1.2e-3 at 16^3 (2e-4 at 8^3): the bounds are those errors
# with a margin.  lambda of D^-1 A does not depend on E or h.
LANCZOS_CASES = [((8, 8, 8), 210.0, 0.45, 2.0, 1e-4), ((16, 8, 8), 7.5, 0.45, 0.125, 1e-4), ((16, 16, 16), 1.0, 0.45, 1.0, 1e-4),
                 ((16, 16, 16), 1.0, 0.3, 1.0 / 16, 1e-5), ((8, 8, 8), 7.5, 0.2, 0.125, 5e-4), ((16, 16, 16), 210.0, 0.2, 2.0, 3e-3)]


@pytest.mark.parametrize("ne,E,nu,h,bound", LANCZOS_CASES)
def test_lanczos_estimate_matches_eigsh_for_materials(ne, E, nu, h, bound):
    import scipy.sparse as sp
    import scipy.sparse.linalg as sla
    A = R.hex_box_csr(ne, (0, 0, 0), ne, E=E, nu=nu, h=h)
    s = sp.diags(1.0 / np.sqrt(A.diagonal()))
    top = sla.eigsh(s @ A @ s, k=1, which="LA", return_eigenvectors=False, tol=1e-14)[0]
    op = G.HexOp(ne, h, nu=nu, E=E)
    assert abs(G.lanczos_lambda(op, 1.0 / op.diag) - top) <= bound * top


@pytest.mark.parametrize("ne", sorted(G.COARSE_SIZES))
def test_coarse_size_boxes_have_the_claimed_coarsest_level(ne):
    lv = G.levels_of(ne)
    assert len(lv) >= 2 and 3 * G.nfree(lv[-1]) == G.COARSE_SIZES[ne]
    assert G.coarsest_matrix(ne, 1.0 / ne[0]).shape == (G.COARSE_SIZES[ne],) * 2


def test_bad_pivot_box_is_indefinite():
    """nu = 0.6 (negative bulk modulus): the coarsest matrix has no Cholesky factor, while the box coarsens normally."""
    assert len(G.levels_of(G.BAD_NU_BOX)) >= 2
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.cholesky(G.coarsest_matrix(G.BAD_NU_BOX, 1.0 / G.BAD_NU_BOX[0], nu=G.BAD_NU))
    np.linalg.cholesky(G.coarsest_matrix(G.BAD_NU_BOX, 1.0 / G.BAD_NU_BOX[0], nu=0.45))


def test_refined_coarse_reference_solves_to_rounding():
    A = G.coarsest_matrix((14, 12, 12), 1.0 / 14, E=210.0, nu=0.45)
    r = np.random.default_rng(5).standard_normal(A.shape[0])
    z = G.refined_solve(A, r)
    res = r.astype(np.longdouble) - A.astype(np.longdouble) @ z.astype(np.longdouble)
    assert float(np.linalg.norm(res.astype(np.float64))) <= 1e-14 * np.linalg.norm(r)


def test_host_vcycle_is_symmetric_positive():
    M = G.HostMultigrid((8, 8, 8), 1.0 / 8)
    rng = np.random.default_rng(2)
    u, v = rng.standard_normal((2, M.A[0].n))
    Mu, Mv = M.apply(u), M.apply(v)
    assert abs(np.dot(Mu, v) - np.dot(u, Mv)) <= 1e-12 * np.linalg.norm(Mu) * np.linalg.norm(v)
    assert np.dot(Mu, u) > 0


@pytest.mark.parametrize("m", [16, 32, 64])
def test_host_vcycle_pcg_iterations_stay_flat(m):
    h = 1.0 / m
    M = G.HostMultigrid((m, m, m), h)
    b = G.load_vector((m, m, m), h)
    x, it = G.pcg(M.A[0], b, M.apply, 1e-8, 50)
    assert it <= 12, it
    assert np.linalg.norm(b - M.A[0] @ x) <= 1e-8 * np.linalg.norm(b)


def test_mg_entry_points_refuse_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pcg_mpi_solver_b200 import _lib
    lib = _lib.load()
    box = _lib.HexBox()
    for a in range(3):
        box.ng[a], box.e0[a], box.ne[a] = 8, 0, 8
    ke = np.zeros(576)
    h = ctypes.c_void_p()
    rc = lib.pcgb_mg_create(None, ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 1.0, 0.125, None, 2, 0.25,
                            ctypes.byref(h))
    assert rc == -4 and b"no CPU fallback" in lib.pcgb_last_error()
    assert lib.pcgb_mg_apply(None, None, None, None) == -4
    assert lib.pcgb_mg_info(None, None, None, None, None) == -4
    assert lib.pcgb_mg_restrict(None, 0, None, None, None) == -4
    assert lib.pcgb_mg_prolong_add(None, 0, None, None, None) == -4
    assert lib.pcgb_mg_smooth(None, 0, None, None, None) == -4
    assert lib.pcgb_mg_coarse_solve(None, None, None, None) == -4
    opt, res = _lib.Options(), _lib.Result()
    assert lib.pcgb_solve_mg(None, None, None, None, None, ctypes.byref(opt), None, ctypes.byref(res), None) == -4
    assert lib.pcgb_mg_destroy(None) == 0
