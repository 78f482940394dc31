"""GPU parity tests of the PCG loop (pcgb_solve through solve()) against the CPU oracle ref_pcg,
which restates pcg_solver.py:356-598 and is pinned to the unmodified reference by the golden tests."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref_pcg as R

pytestmark = pytest.mark.gpu

X_RTOL = 1e-10     # north star: solution/residual parity with the CPU reference to 1e-10 relative
ITER_SLACK = 2     # iteration counts may differ by +-1-2 across summation orders (SURVEY 8(c))


def _oracle(A, b, minv, tol, maxiter, x0=None):
    p = R.CsrPart(A, b, x0=x0)
    return R.ref_pcg([p], [minv], tol, maxiter, exist_dp0=minv is not None)


def test_c1_poisson_matches_oracle(cuda):
    """Config C1: 27-pt Poisson 32^3, b = A x*, x* = rng(0).standard_normal, Jacobi, tol 1e-8."""
    from pcg_mpi_solver_b200 import solve
    A = R.poisson27(32)
    xs = np.random.default_rng(0).standard_normal(A.shape[0])
    b = A @ xs
    minv = 1.0 / A.diagonal()
    ref = _oracle(A, b, minv, 1e-8, 10000)
    x, flag, relres, iters = solve(A, b, minv, 1e-8, 10000)
    assert flag == ref["Flag"] == 0
    assert abs(iters - ref["Iter"]) <= ITER_SLACK
    assert relres <= 1e-8
    # both stop at tol 1e-8: compare at a tolerance where CG itself has converged further
    ref12 = _oracle(A, b, minv, 1e-13, 10000)
    x12, flag12, relres12, _ = solve(A, b, minv, 1e-13, 10000)
    assert flag12 == ref12["Flag"] == 0
    assert np.linalg.norm(x12 - ref12["X"][0]) <= X_RTOL * np.linalg.norm(ref12["X"][0])
    assert abs(relres - ref["RelRes"]) <= 1e-2 * ref["RelRes"] + 1e-12
    # M = "jacobi" builds the same preconditioner on the device (updatePreconditioner, :346-352)
    xj, fj, rj, ij = solve(A, b, "jacobi", 1e-8, 10000)
    assert (fj, ij) == (flag, iters) and np.array_equal(xj, x)


def test_residual_history_matches_oracle(cuda):
    from pcg_mpi_solver_b200 import solve
    A = R.hex_box_csr((8, 8, 8), (0, 0, 0), (8, 8, 8))
    rng = np.random.default_rng(2)
    b = rng.standard_normal(A.shape[0])
    minv = 1.0 / A.diagonal()
    hist = []
    p = R.CsrPart(A, b)
    ref = R.ref_pcg([p], [minv], 1e-9, 5000, resvec=hist)
    x, flag, relres, iters, info = solve(A, b, minv, 1e-9, 5000, record_resvec=True, return_info=True)
    assert flag == ref["Flag"] == 0 and abs(iters - ref["Iter"]) <= ITER_SLACK
    # CG residual histories of two fp64 implementations agree to rounding at first and then drift apart
    # (loss of orthogonality amplifies summation-order differences): tight early, loose later
    m = min(len(hist), len(info.resvec)) - 1  # the last entry is the verified residual on the oracle side
    np.testing.assert_allclose(info.resvec[:12], np.array(hist[:12]), rtol=1e-9)
    np.testing.assert_allclose(info.resvec[:m], np.array(hist[:m]), rtol=0.5)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("check_every", [1, 7, 64])
def test_batching_is_exact(cuda, use_graph, check_every):
    """The device-side state machine stops at the same iteration whatever the host polling period."""
    from pcg_mpi_solver_b200 import solve
    A = R.poisson27(12)
    b = A @ np.random.default_rng(4).standard_normal(A.shape[0])
    minv = 1.0 / A.diagonal()
    base = solve(A, b, minv, 1e-10, 1000, check_every=1, use_graph=False)
    got = solve(A, b, minv, 1e-10, 1000, check_every=check_every, use_graph=use_graph)
    assert got[1:] == base[1:]
    assert np.array_equal(got[0], base[0])


def test_no_preconditioner_and_x0(cuda):
    from pcg_mpi_solver_b200 import solve
    A = R.poisson27(10)
    rng = np.random.default_rng(7)
    b = A @ rng.standard_normal(A.shape[0])
    x0 = rng.standard_normal(A.shape[0])
    ref = _oracle(A, b, None, 1e-9, 1000, x0=x0)
    x, flag, relres, iters = solve(A, b, None, 1e-9, 1000, x0=x0)
    assert flag == ref["Flag"] == 0 and abs(iters - ref["Iter"]) <= ITER_SLACK and relres <= 1e-9


def test_flag1_maxiter_returns_xmin(cuda):
    """Non-converged path (:568-584): flag 1, Iter/RelRes from the min-residual bookkeeping, x = XMin."""
    from pcg_mpi_solver_b200 import solve
    A = R.hex_box_csr((6, 6, 6), (0, 0, 0), (6, 6, 6))
    b = np.random.default_rng(8).standard_normal(A.shape[0])
    minv = 1.0 / A.diagonal()
    for maxiter in (1, 5, 23):
        ref = _oracle(A, b, minv, 1e-12, maxiter)
        x, flag, relres, iters = solve(A, b, minv, 1e-12, maxiter)
        assert flag == ref["Flag"] == 1
        # while XMin is still bound to X (no improvement recorded, :379-380) Iter hangs on a rounding-level comparison
        assert iters == ref["Iter"] or (ref["aliased"] and iters in (1, maxiter))
        assert abs(relres - ref["RelRes"]) <= 1e-9 * ref["RelRes"]
        assert np.linalg.norm(x - ref["X"][0]) <= 1e-9 * np.linalg.norm(ref["X"][0])


@pytest.mark.parametrize("case", ["maxiter3", "maxiter30"])
def test_maxiter_exit_matches_reference_golden(cuda, tmp_path, case):
    """Non-converged exit against the UNMODIFIED reference (tests/golden/hex_maxiter_ref.*, oracle/make_golden_maxiter.py):
    maxiter3 = the residual is still growing, MP_XMin is still the same array as MP_X (pcg_solver.py:379-380, :516) and
    the reference exports the LATEST iterate; maxiter30 = XMin is the frozen minimum-residual copy (:555-558)."""
    import json
    import os
    from oracle.hex_mdf import write_hex_mdf
    from pcg_mpi_solver_b200 import solve
    from pcg_mpi_solver_b200.model import load_mdf
    from pcg_mpi_solver_b200.partition import build_subdomains
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    meta = json.load(open(os.path.join(gold, "hex_maxiter_ref.json")))
    arr = np.load(os.path.join(gold, "hex_maxiter_ref.npz"))
    run = meta["runs"][case]
    write_hex_mdf(str(tmp_path), tuple(meta["ng"]))
    model = load_mdf(str(tmp_path), name="hexmodel")
    sub = build_subdomains(model, np.zeros(model.n_elem, dtype=np.int64), 1, assemble=True)[0]
    x, flag, relres, iters = solve(sub.A, sub.b, 1.0 / sub.A.diagonal(), meta["tol"], run["maxiter"])
    assert flag == run["Flag"] == 1
    assert iters in ((run["Iter"], 1) if case == "maxiter3" else (run["Iter"],))
    assert abs(relres - run["RelRes"]) <= 1e-9 * run["RelRes"]
    u = np.zeros(model.n_dof)
    u[sub.dof_eff_global] = x
    uref = arr[f"U_{case}"]
    assert np.linalg.norm(u - uref) <= 1e-11 * np.linalg.norm(uref)


def test_early_exits(cuda):
    from pcg_mpi_solver_b200 import solve
    A = R.poisson27(6)
    n = A.shape[0]
    x0 = np.random.default_rng(9).standard_normal(n)
    # zero right-hand side: the reference returns the INITIAL GUESS, flag 0, relres 0, iter 0 (:387-395)
    x, flag, relres, iters = solve(A, np.zeros(n), None, 1e-8, 100, x0=x0)
    assert (flag, relres, iters) == (0, 0.0, 0) and np.array_equal(x, x0)
    # initial guess already good enough (:421-426)
    b = A @ x0
    x, flag, relres, iters = solve(A, b, None, 1e-6, 100, x0=x0)
    assert flag == 0 and iters == 0 and relres <= 1e-6 and np.array_equal(x, x0)


def test_breakdown_flags(cuda):
    from pcg_mpi_solver_b200 import solve
    n = 50
    rng = np.random.default_rng(10)
    b = rng.standard_normal(n)
    # flag 4: indefinite operator -> p.q <= 0 (:492-494)
    A = sp.diags(np.concatenate([np.ones(n // 2), -np.ones(n - n // 2)])).tocsr()
    ref = _oracle(A, b, None, 1e-10, 100)
    x, flag, relres, iters = solve(A, b, None, 1e-10, 100)
    assert flag == ref["Flag"] == 4 and iters == ref["Iter"]
    # flag 2: infinite preconditioner entry (:448-450)
    A = sp.diags(np.linspace(1, 2, n)).tocsr()
    minv = np.ones(n)
    minv[3] = np.inf
    ref = _oracle(A, b, minv, 1e-10, 100)
    x, flag, relres, iters = solve(A, b, minv, 1e-10, 100)
    assert flag == ref["Flag"] == 2 and iters == ref["Iter"]


def test_too_small_tolerance_flag3(cuda):
    """tol below what fp64 can deliver: either stagnation (:560-562) or the verification step keeps failing
    until MoreSteps reaches MaxMSteps, where the reference raises Warning('PCG : TooSmallTolerance')
    (:548-549); MATLAB semantics (and ours) = flag 3.  Which of the two fires depends on rounding, so a
    few tolerances are tried and the raise path is exercised wherever the device reports it."""
    from pcg_mpi_solver_b200 import solve
    A = R.poisson27(8)
    b = A @ np.random.default_rng(11).standard_normal(A.shape[0])
    minv = 1.0 / A.diagonal()
    seen_too_small = False
    for tol in (1e-16, 3e-17, 1e-17, 1e-18):
        ref = _oracle(A, b, minv, tol, 400)
        x, flag, relres, iters, info = solve(A, b, minv, tol, 400, return_info=True)
        assert ref["Flag"] == 3 and flag == 3
        assert abs(iters - ref["Iter"]) <= 6
        assert relres < 1e-14
        if info.too_small_tol:
            seen_too_small = True
            assert info.moresteps >= 5
            with pytest.raises(Warning):
                solve(A, b, minv, tol, 400, on_too_small_tol="raise")
    # MaxMSteps = min(n/50, 5, n - maxiter) (:404): maxiter > n makes it negative -> first failed check aborts
    x, flag, relres, iters, info = solve(A, b, minv, 1e-17, 2000, return_info=True)
    ref = _oracle(A, b, minv, 1e-17, 2000)
    assert flag == ref["Flag"] == 3 and info.too_small_tol and ref["too_small_tol"]
    seen_too_small = True
    assert seen_too_small


def test_hex_generator_matches_oracle_assembly(cuda):
    """csrc/hexgen.cuh against plain scipy assembly of the same box (incl. an interior, unclamped box)."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    for ng, e0, ne in [((5, 4, 3), (0, 0, 0), (5, 4, 3)), ((8, 6, 4), (4, 0, 2), (4, 3, 2)), ((3, 3, 3), (1, 1, 1), (1, 1, 1))]:
        M = generate_matrix(HexBlock(ng, e0, ne), device=cuda).to_scipy()
        A = R.hex_box_csr(ng, e0, ne)
        assert M.shape == A.shape and M.nnz == A.nnz
        assert np.array_equal(M.indptr, A.indptr) and np.array_equal(M.indices, A.indices)
        np.testing.assert_allclose(M.data, A.data, rtol=1e-13, atol=1e-15)


# (ng, e0, ne, material): boxes one element thick on each axis, on the clamped x = 0 face (nx = 1 there leaves one free node
# layer) and away from it, and non-default E, nu, h
HEX_BOXES = [
    ((4, 3, 3), (0, 0, 0), (1, 3, 3), {}),
    ((4, 3, 3), (2, 0, 0), (1, 3, 3), {}),
    ((4, 3, 3), (0, 1, 0), (2, 1, 3), {}),
    ((4, 3, 3), (1, 2, 0), (3, 1, 3), {}),
    ((4, 3, 3), (0, 0, 2), (4, 3, 1), {}),
    ((4, 3, 3), (1, 0, 1), (2, 3, 1), {}),
    ((1, 1, 1), (0, 0, 0), (1, 1, 1), {}),
    ((3, 3, 3), (1, 1, 1), (1, 1, 1), dict(E=7.5, nu=0.2, h=0.25)),
    ((5, 4, 3), (0, 0, 0), (5, 4, 3), dict(E=210.0, nu=0.25, h=0.125)),
    ((6, 4, 4), (2, 1, 1), (3, 2, 2), dict(E=3.5, nu=0.45, h=2.0)),
]


@pytest.mark.parametrize("ng, e0, ne, mat", HEX_BOXES)
def test_hex_generator_thin_boxes_and_materials(cuda, ng, e0, ne, mat):
    """csrc/hexgen.cuh against plain scipy assembly on thin boxes and other materials: structure exact."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    M = generate_matrix(HexBlock(ng, e0, ne, **mat), device=cuda).to_scipy()
    A = R.hex_box_csr(ng, e0, ne, **mat)
    assert M.shape == A.shape and M.nnz == A.nnz
    assert np.array_equal(M.indptr, A.indptr) and np.array_equal(M.indices, A.indices)
    np.testing.assert_allclose(M.data, A.data, rtol=1e-13, atol=1e-15 * np.abs(A.data).max())


def test_hex_solve_c2_small(cuda):
    """A small instance of config C2 end to end on the device generator + solve."""
    import torch
    from pcg_mpi_solver_b200 import solve
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock((16, 16, 16), (0, 0, 0), (16, 16, 16), h=1.0 / 16)
    A = generate_matrix(blk, device=cuda)
    op = SubdomainOperator(A)
    b = load_vector(blk, device=cuda)
    minv = op.jacobi()
    x, flag, relres, iters = solve(op, b, minv, 1e-9, 5000)
    As = R.hex_box_csr(blk.ng, blk.e0, blk.ne, h=blk.h)
    ref = _oracle(As, b.cpu().numpy(), 1.0 / As.diagonal(), 1e-9, 5000)
    assert flag == ref["Flag"] == 0 and abs(iters - ref["Iter"]) <= ITER_SLACK
    r = b.cpu().numpy() - As @ x.cpu().numpy()
    assert np.linalg.norm(r) <= 1e-9 * np.linalg.norm(b.cpu().numpy()) * (1 + 1e-6)
    ref13 = _oracle(As, b.cpu().numpy(), 1.0 / As.diagonal(), 1e-13, 5000)
    x13 = solve(op, b, minv, 1e-13, 5000)[0]
    assert np.linalg.norm(x13.cpu().numpy() - ref13["X"][0]) <= 1e-9 * np.linalg.norm(ref13["X"][0])


def test_two_host_threads_two_solvers(cuda):
    """Re-entrancy of the C ABI (SURVEY 8(b): "re-entrant per handle, no global state besides last-error TLS"): two host threads,
    each with its own matrix / solver handle (ctypes releases the GIL during the calls), solve different systems at the
    same time; results are bit-identical to the same solves run one after the other.  pcgb_dot_w (stream-ordered scratch) too."""
    import threading

    import torch
    from pcg_mpi_solver_b200 import _lib, solve
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    systems = []
    for seed, A in ((1, R.hex_box_csr((10, 8, 6), (0, 0, 0), (10, 8, 6))), (2, R.poisson27(14))):
        b = np.random.default_rng(seed).standard_normal(A.shape[0])
        systems.append((A, b, 1.0 / A.diagonal()))
    serial = [solve(A, b, m, 1e-11, 3000) for A, b, m in systems]
    ops = [SubdomainOperator(CsrMatrix.from_scipy(A, device=cuda)) for A, _, _ in systems]
    out, errs = [None, None], []

    def work(k):
        try:
            A, b, m = systems[k]
            s = torch.cuda.Stream(device=cuda)
            with torch.cuda.stream(s):
                bd, md = torch.from_numpy(b).to(cuda), torch.from_numpy(m).to(cuda)
                for _ in range(5):                                   # several solves per thread: graphs, buffers and scratch are per handle
                    x, info = ops[k].solve(bd, md, 1e-11, 3000)
                d = torch.zeros(1, dtype=torch.float64, device=cuda)
                _lib.check(_lib.load().pcgb_dot_w(bd.numel(), _lib.ptr(bd), _lib.ptr(bd), None, _lib.ptr(d), s.cuda_stream))
                s.synchronize()
                out[k] = (x.cpu().numpy(), info.flag, info.relres, info.iters, float(d))
        except Exception as e:  # pragma: no cover
            errs.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errs, errs
    for k in range(2):
        x, flag, relres, iters, d = out[k]
        assert (flag, relres, iters) == serial[k][1:] and np.array_equal(x, serial[k][0])
        assert abs(d - float(systems[k][1] @ systems[k][1])) <= 1e-12 * d
