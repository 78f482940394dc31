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
