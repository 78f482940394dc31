"""The geometric multigrid preconditioner (csrc/gmg.cuh, pcgb_mg_*, multigrid.HexMultigrid): transfers entrywise against a
long-double gather, the smoother, eigenvalue estimates and coarse solve against the host restatement (tests/gmg_cases.py),
the whole V-cycle, and MG-PCG solves with every exit of the loop, trace replay and refusals."""
import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import gmg_cases as G
from tests import pcg_shadow as S

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -53


def _setup(cuda, ne, kind="csr", degree=2, lo=0.25):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock(tuple(ne), (0, 0, 0), tuple(ne), h=1.0 / ne[0])
    A = generate_matrix(blk, device=cuda) if kind == "csr" else generate_ebe(blk, device=cuda, ordered=kind == "ebe_ordered")
    op = SubdomainOperator(A)
    return blk, op, HexMultigrid(op, blk, degree=degree, lo=lo)


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


@pytest.mark.parametrize("ne", [(4, 4, 4), (4, 8, 16), (16, 8, 4), (80, 80, 48), (80, 80, 64)])
def test_transfers_entrywise(cuda, ne):
    """Restriction (<= 27 terms) and prolongation-add (<= 8 terms + x) within (k+2) 2^-53 sum|terms| of a long-double gather
    in the same order; boxes with 2 elements per axis on the coarse level, non-cubic boxes, lengths around the vector-grid cap."""
    _, _, mg = _setup(cuda, ne)
    rng = np.random.default_rng(sum(ne))
    n = mg.info()["n"]
    rf = rng.standard_normal(n[0])
    rc = mg.restrict(0, _t(rf, cuda)).cpu().numpy()
    ref, mag = G.restrict(rf, ne, np.longdouble)
    assert np.all(np.abs(rc - ref) <= (27 + 2) * EPS * mag)
    ec, xf = rng.standard_normal(n[1]), rng.standard_normal(n[0])
    out = mg.prolong_add(0, _t(ec, cuda), _t(xf, cuda)).cpu().numpy()
    ref, mag = G.prolong_add(ec, xf, ne, np.longdouble)
    assert np.all(np.abs(out - ref) <= (9 + 2) * EPS * mag)


@pytest.mark.parametrize("m", [16, 32])
def test_lambda_estimates_and_smoother(cuda, m):
    """lambda within 5 % of eigsh on every smoothed level; one smoothing x += S(b - A x) from x = 0 and from x != 0 equals the
    host restatement fed the device's lambda to 1e-13, on the fine (solver operator) and a coarse (generated CSR) level."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as sla
    _, _, mg = _setup(cuda, (m, m, m))
    info = mg.info()
    H = G.HostMultigrid((m, m, m), 1.0 / m, lambdas=info["lambda"])
    for l in range(info["levels"] - 1):
        A = R.hex_box_csr(H.ne[l], (0, 0, 0), H.ne[l], h=2.0 ** l / m)
        s = sp.diags(1.0 / np.sqrt(A.diagonal()))
        top = sla.eigsh(s @ A @ s, k=1, which="LA", return_eigenvectors=False)[0]
        assert abs(info["lambda"][l] - top) <= 0.05 * top, (l, info["lambda"][l], top)
    rng = np.random.default_rng(m)
    for l in (0, 1):
        b, x0 = rng.standard_normal(info["n"][l]), rng.standard_normal(info["n"][l])
        for start in (np.zeros_like(x0), x0):
            x = mg.smooth(l, _t(b, cuda), _t(start, cuda)).cpu().numpy()
            ref, _ = H.smooth(l, b, start, False)
            assert np.linalg.norm(x - ref) <= 1e-13 * np.linalg.norm(ref), l


def test_coarse_solve(cuda):
    _, _, mg = _setup(cuda, (16, 8, 8))
    nec = G.levels_of((16, 8, 8))[-1]
    Ac = R.hex_box_csr(nec, (0, 0, 0), nec, h=2.0 ** (len(G.levels_of((16, 8, 8))) - 1) / 16)
    r = np.random.default_rng(3).standard_normal(Ac.shape[0])
    z = mg.coarse_solve(_t(r, cuda)).cpu().numpy()
    assert np.linalg.norm(Ac @ z - r) <= 1e-12 * np.linalg.norm(r)


def test_coarse_limit_and_refusals_leak_nothing(cuda):
    """A coarsest level of 1536 dofs is built and solves, and destroying it gives back all device memory it took; the next
    possible size (1539: dofs come in threes) is refused, as are a multi-rank solver, an odd ne, e0 != 0, degree < 1 and lo
    outside (0, 1.1) or NaN - all before anything is allocated."""
    import gc
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk, op, mg = _setup(cuda, (16, 14, 14))
    info = mg.info()
    assert info["n"][-1] == 1536 and info["levels"] == 2
    A = R.hex_box_csr((8, 7, 7), (0, 0, 0), (8, 7, 7), h=2.0 / 16)
    r = np.random.default_rng(4).standard_normal(1536)
    assert np.linalg.norm(A @ mg.coarse_solve(_t(r, cuda)).cpu().numpy() - r) <= 1e-12 * np.linalg.norm(r)
    del mg
    gc.collect()
    # a second hierarchy on the same operator (kernels are loaded by now): device memory before create == after destroy
    minv = op.jacobi()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0, _ = torch.cuda.mem_get_info(cuda)
    mg = HexMultigrid(op, blk, minv=minv)
    assert torch.cuda.mem_get_info(cuda)[0] < free0
    mg = None
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info(cuda)[0] >= free0

    def refused(blk_, op_, **kw):
        torch.cuda.synchronize()
        free0, _ = torch.cuda.mem_get_info(cuda)
        with pytest.raises(_lib.PcgbError, match=r"\(-1\)"):
            HexMultigrid(op_, blk_, **kw)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info(cuda)[0] >= free0

    big = HexBlock((38, 4, 16), (0, 0, 0), (38, 4, 16), h=1.0 / 38)
    assert 3 * G.nfree(G.levels_of(big.ne)[-1]) == 1539
    refused(big, SubdomainOperator(generate_matrix(big, device=cuda)))
    odd = HexBlock((16, 16, 15), (0, 0, 0), (16, 16, 15), h=1.0 / 16)
    refused(odd, SubdomainOperator(generate_matrix(odd, device=cuda)))
    off = HexBlock((32, 16, 16), (16, 0, 0), (16, 16, 16), h=1.0 / 32)
    refused(off, SubdomainOperator(generate_matrix(off, device=cuda)))
    refused(blk, op, degree=0)
    for lo in (0.0, 1.1, float("nan")):     # the Chebyshev interval [lo, 1.1] lambda must be non-empty and positive
        refused(blk, op, lo=lo)
    # a solver with a communicator (one peer-only rank stands for a multi-rank solver)
    from pcg_mpi_solver_b200.solver import Communicator
    comm = Communicator(0, 1, None, device=cuda)
    refused(blk, SubdomainOperator(op.A, comm=comm))


@pytest.mark.parametrize("kind", ["csr", "ebe_ordered", "ebe"])
def test_vcycle_matches_host_symmetric_and_reproducible(cuda, kind):
    import torch
    ne = (16, 16, 16)
    _, _, mg = _setup(cuda, ne, kind)
    H = G.HostMultigrid(ne, 1.0 / 16, lambdas=mg.info()["lambda"])
    rng = np.random.default_rng(6)
    u, v = rng.standard_normal((2, mg.n))
    Mu, Mv = mg.apply(_t(u, cuda)).cpu().numpy(), mg.apply(_t(v, cuda)).cpu().numpy()
    ref = H.apply(u)
    assert np.linalg.norm(Mu - ref) <= 1e-12 * np.linalg.norm(ref)
    assert abs(np.dot(Mu, v) - np.dot(u, Mv)) <= 1e-12 * np.linalg.norm(Mu) * np.linalg.norm(v)
    for w in rng.standard_normal((4, mg.n)):
        assert np.dot(mg.apply(_t(w, cuda)).cpu().numpy(), w) > 0
    if kind != "ebe":   # the atomic EBE operator is not bit-reproducible
        a, b = mg.apply(_t(u, cuda)), mg.apply(_t(u, cuda))
        assert torch.equal(a, b) and np.array_equal(a.cpu().numpy(), Mu)


@pytest.mark.parametrize("m", [16, 32, 64])
def test_solve_iterations_and_solution(cuda, m):
    """Flag 0 within +-1 of the host restatement's count and <= 12 iterations; x against Jacobi-PCG at tol 1e-12."""
    from pcg_mpi_solver_b200 import solve
    from pcg_mpi_solver_b200.hexmesh import load_vector
    blk, op, mg = _setup(cuda, (m, m, m))
    b = load_vector(blk, device=cuda)
    x, flag, relres, iters = solve(op, b, mg, 1e-8, 100)
    H = G.HostMultigrid((m, m, m), 1.0 / m, lambdas=mg.info()["lambda"])
    _, host_iters = G.pcg(H.A[0], b.cpu().numpy(), H.apply, 1e-8, 100)
    assert flag == 0 and iters <= 12 and abs(iters - host_iters) <= 1, (iters, host_iters)
    x12, flag12, _, it12 = solve(op, b, mg, 1e-12, 100)
    assert flag12 == 0
    if m <= 32:   # Jacobi-PCG stagnates before 1e-12 on 64^3 (flag 3)
        xj, flagj, _, _ = solve(op, b, "jacobi", 1e-12, 20000)
        assert flagj == 0 and (x12 - xj).norm() <= 1e-9 * xj.norm()


def test_solves_bit_identical_across_graph_and_batching_and_trace_replays(cuda):
    import torch
    from pcg_mpi_solver_b200.hexmesh import load_vector
    blk, op, mg = _setup(cuda, (16, 16, 16), "ebe_ordered")
    b = load_vector(blk, device=cuda)
    base, info0 = op.solve(b, mg, 1e-12, 200, trace=True, check_every=1, use_graph=False, record_resvec=True)
    assert info0.flag == 0
    sh = S.replay(info0.trace, 1e-12, 200, mg.n)
    assert sh.result["flag"] == info0.flag
    for use_graph in (False, True):
        for check_every in (1, 7, 200):
            x, info = op.solve(b, mg, 1e-12, 200, trace=True, check_every=check_every, use_graph=use_graph, record_resvec=True)
            assert torch.equal(x, base), (use_graph, check_every)
            assert info.trace.tobytes() == info0.trace.tobytes() and np.array_equal(info.resvec, info0.resvec)


def test_exits(cuda):
    """maxiter (flag 1), b = 0, x0 given or omitted, NaN in the fine Minv (flag 2)."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blk, op, mg = _setup(cuda, (16, 8, 8))
    b = load_vector(blk, device=cuda)
    x, info = op.solve(b, mg, 1e-14, 3)
    assert info.flag == 1 and info.iters <= 3
    x, info = op.solve(torch.zeros_like(b), mg, 1e-8, 50)
    assert info.flag == 0 and info.iters == 0 and not x.any()
    x0 = torch.from_numpy(np.random.default_rng(1).standard_normal(mg.n)).to(cuda)
    xa, ia = op.solve(b, mg, 1e-10, 50, x0=x0)
    xb, ib = op.solve(b, mg, 1e-10, 50)
    assert ia.flag == ib.flag == 0 and (xa - xb).norm() <= 1e-8 * xb.norm()
    minv = op.jacobi()
    minv[5] = float("nan")
    bad = HexMultigrid(op, blk, minv=minv)
    x, info = op.solve(b, bad, 1e-8, 50)
    assert info.flag == 2


def test_destroying_a_handle_drops_the_solver_graph(cuda):
    """Solve with graphs on, destroy the handle, build a degree-3 handle on the same operator (malloc usually hands back the
    same address, so the graph key alone cannot tell them apart): the graphed solve equals a direct-launch solve, x and trace."""
    import gc
    import torch
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blk, op, mg = _setup(cuda, (16, 16, 16))
    b = load_vector(blk, device=cuda)
    x2, info2 = op.solve(b, mg, 1e-10, 200, use_graph=True, check_every=4)
    assert info2.flag == 0
    del mg
    gc.collect()
    mg3 = HexMultigrid(op, blk, degree=3)
    xg, ig = op.solve(b, mg3, 1e-10, 200, use_graph=True, check_every=4, trace=True)
    xd, idr = op.solve(b, mg3, 1e-10, 200, use_graph=False, check_every=4, trace=True)
    assert ig.flag == idr.flag == 0 and ig.iters == idr.iters
    assert torch.equal(xg, xd) and ig.trace.tobytes() == idr.trace.tobytes()
    assert not torch.equal(xg, x2)   # degree 3 is a different preconditioner
