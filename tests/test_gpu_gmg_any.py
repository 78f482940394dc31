"""HexMultigrid(coarsening="any") on the device (pcgb_mg_create_any): the level boxes against the rule, every smoothed level
against scipy P^T A P, the transfers against the host P on levels with odd and kept axes, the smoother and V-cycle against
the host restatement (tests/gmg_any_cases.py), bit-identity with the default field hierarchy where both coincide, MG-PCG on
boxes the default refuses, launches per iteration and refusals."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp

from tests import gmg_any_cases as A
from tests import gmg_cases as G
from tests import voxel_cases as V

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -53

# fine box -> (host MG-PCG iterations at contrast 1, at contrast 100), tol 1e-8, degree 2, b = hexmesh.load_vector
PINNED = {(25, 25, 25): (23, 66), (38, 4, 16): (18, 127), (33, 33, 33): (26, 83)}


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _setup(cuda, ne, field=None, kind="csr", degree=2, coarsening="any", E=1.0):
    """(block, operator, preconditioner) of the whole box ne, h = 1 / ne[0]; field None: uniform E."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0], E=E)
    M = generate_matrix(blk, device=cuda, E_field=field) if kind == "csr" else \
        generate_ebe(blk, device=cuda, ordered=kind == "ebe_ordered", E_field=field)
    op = SubdomainOperator(M)
    return blk, op, HexMultigrid(op, blk, degree=degree, E_field=field, coarsening=coarsening)


def _field(ne, which, seed=0):
    return np.ones((ne[2], ne[1], ne[0])) if which == "uniform" else V.two_phase(ne, 100.0, seed=seed)


def _dev_csr(mg, l, shape):
    rp, col, val = mg.level_matrix(l)
    return sp.csr_matrix((val.cpu().numpy(), col.cpu().numpy(), rp.cpu().numpy()), shape=shape)


BOXES = [((16, 16, 15), "uniform"), ((16, 16, 15), "inclusion"), ((38, 4, 16), "uniform"), ((38, 4, 16), "inclusion"),
         ((8, 8, 5), "inclusion"), ((25, 17, 9), "uniform"), ((25, 17, 9), "inclusion"), ((31, 31, 31), "uniform"),
         ((31, 31, 31), "inclusion")]


@pytest.mark.parametrize("ne,which", BOXES)
def test_levels_equal_ptap(cuda, ne, which):
    """level_shapes() is the rule's; every smoothed level is exactly symmetric and equal to scipy P^T A P of the fine voxel
    matrix within 1e-12 of the row's largest entry; the coarsest solve matches a dense solve of P^T A P.  A uniform box
    passes no field (Ck = E h inside the library)."""
    f = _field(ne, which, seed=sum(ne))
    blk, op, mg = _setup(cuda, ne, None if which == "uniform" else f)
    lv = A.levels(ne)
    assert mg.level_shapes() == lv
    info = mg.info()
    assert info["levels"] == len(lv) and info["n"] == [3 * G.nfree(n_) for n_ in lv]
    mats = A.ptap_matrices(f, blk.h)
    for l in range(1, len(lv) - 1):
        D = _dev_csr(mg, l, mats[l].shape)
        assert (D != D.T).nnz == 0
        diff = abs(D - mats[l]).max(axis=1).toarray().ravel()
        rowmax = abs(mats[l]).max(axis=1).toarray().ravel()
        assert np.all(diff <= 1e-12 * rowmax), (l, float(np.max(diff / rowmax)))
    Ac = mats[-1].toarray()
    r = np.random.default_rng(3).standard_normal(Ac.shape[0])
    z = mg.coarse_solve(_t(r, cuda)).cpu().numpy()
    zr = G.refined_solve(Ac, r)
    assert np.linalg.norm(z - zr) <= 1e-10 * np.linalg.norm(zr)
    s = mg.setup_info()
    ncell = [int(np.prod(n_)) for n_ in lv]
    assert s["galerkin_ms"] > 0
    assert s["element_matrix_peak_bytes"] == max(4608 * (ncell[l] + (ncell[l - 1] if l > 1 else 0)) for l in range(1, len(lv)))


@pytest.mark.parametrize("ne", [(16, 16, 15), (38, 4, 16), (8, 8, 5), (25, 17, 9), (31, 31, 31), (1, 5, 9)])
def test_transfers_match_host_P(cuda, ne):
    """restrict / prolong_add on every level against the host P (levels with odd axes, kept axes and the clamped plane):
    each entry within (k + 2) 2^-53 of the sum of |terms|, where k <= 27 is the number of terms."""
    f = _field(ne, "inclusion", seed=1)
    _, _, mg = _setup(cuda, ne, f)
    lv = A.levels(ne)
    rng = np.random.default_rng(5)
    for l in range(len(lv) - 1):
        P = A.prolongation_any(lv[l])
        rf = rng.standard_normal(P.shape[0])
        rc = mg.restrict(l, _t(rf, cuda)).cpu().numpy()
        ref, mag = P.T @ rf, abs(P.T) @ np.abs(rf)
        assert np.all(np.abs(rc - ref) <= 29 * EPS * mag), l
        ec, xf = rng.standard_normal(P.shape[1]), rng.standard_normal(P.shape[0])
        got = mg.prolong_add(l, _t(ec, cuda), _t(xf, cuda)).cpu().numpy()
        ref, mag = xf + P @ ec, np.abs(xf) + abs(P) @ np.abs(ec)
        assert np.all(np.abs(got - ref) <= 10 * EPS * mag), l


@pytest.mark.parametrize("kind", ["csr", "ebe_ordered", "ebe"])
@pytest.mark.parametrize("degree", [1, 2, 3])
@pytest.mark.parametrize("ne", [(25, 17, 9), (38, 4, 16)])
def test_vcycle_parts_match_host(cuda, kind, degree, ne):
    """lambda per level against the host Lanczos on the host levels (1e-10); fed the device's lambda and D^-1: one smoothing
    per level (1e-12), the whole V-cycle (1e-12) and its symmetry (1e-12)."""
    f = _field(ne, "inclusion", seed=7)
    blk, op, mg = _setup(cuda, ne, f, kind, degree=degree)
    info = mg.info()
    mats = A.level_matrices(f, blk.h)
    H0 = A.HostAnyMultigrid(f, blk.h, degree=degree, mats=mats)
    lam = info["lambda"][:info["levels"] - 1]
    assert np.allclose(lam, H0.lam, rtol=1e-10, atol=0), (lam, H0.lam)
    H = A.HostAnyMultigrid(f, blk.h, degree=degree, lambdas=lam, minv=op.jacobi().cpu().numpy(), mats=mats)
    rng = np.random.default_rng(degree)
    for l in range(info["levels"] - 1):
        b, x0 = rng.standard_normal(info["n"][l]), rng.standard_normal(info["n"][l])
        x = mg.smooth(l, _t(b, cuda), _t(x0, cuda)).cpu().numpy()
        ref, _ = H.smooth(l, b, x0, False)
        assert np.linalg.norm(x - ref) <= 1e-12 * np.linalg.norm(ref), l
    u, v = rng.standard_normal((2, mg.n))
    Mu, Mv = mg.apply(_t(u, cuda)).cpu().numpy(), mg.apply(_t(v, cuda)).cpu().numpy()
    ref = H.apply(u)
    assert np.linalg.norm(Mu - ref) <= 1e-12 * np.linalg.norm(ref)
    assert abs(np.dot(Mu, v) - np.dot(u, Mv)) <= 1e-12 * np.linalg.norm(Mu) * np.linalg.norm(v)


def test_even_box_bit_identical_to_field_path(cuda):
    """On 32^3 with a field both hierarchies are the same: identical level matrices, lambda, V-cycle and MG-PCG x."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    ne = (32, 32, 32)
    f = V.two_phase(ne, 100.0, seed=32)
    blk, op, mg = _setup(cuda, ne, f)
    ev = HexMultigrid(op, blk, E_field=f)
    assert mg.level_shapes() == ev.level_shapes() and mg.info()["lambda"] == ev.info()["lambda"]
    for l in range(1, mg.info()["levels"] - 1):
        assert all(torch.equal(a, b) for a, b in zip(mg.level_matrix(l), ev.level_matrix(l))), l
    r = _t(np.random.default_rng(1).standard_normal(mg.n), cuda)
    assert torch.equal(mg.apply(r), ev.apply(r))
    b = load_vector(blk, device=cuda)
    xa, ia = op.solve(b, mg, 1e-8, 200)
    xe, ie = op.solve(b, ev, 1e-8, 200)
    assert ia.flag == 0 and ia.iters == ie.iters and torch.equal(xa, xe)


def test_shared_levels_identical_then_continue(cuda):
    """Where the default field path stops (16x14x14 -> 8x7x7, 32x28x28 -> 16x14x14 -> 8x7x7), "any" has the same levels
    bit for bit and continues below 8x7x7 to 4x4x4 and 2x2x2."""
    import torch
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    for ne in ((16, 14, 14), (32, 28, 28)):
        f = V.random_field(ne, seed=ne[0])
        blk, op, mg = _setup(cuda, ne, f)
        ev = HexMultigrid(op, blk, E_field=f)
        se, sa = ev.level_shapes(), mg.level_shapes()
        assert se[-1] == (8, 7, 7) and sa == se + [(4, 4, 4), (2, 2, 2)]
        k = len(se)
        assert mg.info()["lambda"][:k - 1] == ev.info()["lambda"][:k - 1]
        for l in range(1, k - 1):
            assert all(torch.equal(a, b) for a, b in zip(mg.level_matrix(l), ev.level_matrix(l))), (ne, l)
        rng = np.random.default_rng(2)
        for l in range(k - 1):
            x, y = _t(rng.standard_normal(mg.info()["n"][l + 1]), cuda), _t(rng.standard_normal(mg.info()["n"][l]), cuda)
            assert torch.equal(mg.restrict(l, y), ev.restrict(l, y))
            assert torch.equal(mg.prolong_add(l, x, y.clone()), ev.prolong_add(l, x, y.clone()))


@pytest.mark.parametrize("ne,contrast", [((25, 25, 25), 1), ((25, 25, 25), 100), ((33, 33, 33), 1), ((33, 33, 33), 100),
                                         ((38, 4, 16), 1), ((38, 4, 16), 100), ((50, 40, 30), 1), ((50, 40, 30), 100),
                                         ((100, 100, 100), 1)])
def test_mg_pcg_on_boxes_the_default_refuses(cuda, ne, contrast):
    """The default coarsening refuses each box; "any" reaches 1e-8 (within 2 of the pinned host count where pinned), and its
    1e-11 solution, refined once by an MG-PCG solve of its residual, agrees with a sparse direct solve (small boxes) or 1e-13
    Jacobi-PCG to 1e-9 (a solve may stagnate, flag 3, just above its tolerance)."""
    import torch
    import scipy.sparse.linalg as sla
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    if ne == (100, 100, 100) and torch.cuda.mem_get_info(cuda)[0] < 8e9:
        pytest.skip("needs ~8 GB of free device memory")
    f = None if contrast == 1 else V.two_phase(ne, contrast, seed=0)
    blk, op, mg = _setup(cuda, ne, f)
    with pytest.raises(_lib.PcgbError):
        HexMultigrid(op, blk, E_field=f)
    b = load_vector(blk, device=cuda)
    x, info = op.solve(b, mg, 1e-8, 300)
    assert info.flag == 0, (info.flag, info.iters)
    if ne in PINNED:
        want = PINNED[ne][0 if contrast == 1 else 1]
        assert abs(info.iters - want) <= 2, (info.iters, want)
    x11, i11 = op.solve(b, mg, 1e-11, 800)
    assert i11.flag in (0, 3) and i11.relres <= 1e-10, (i11.flag, i11.relres)
    r = b - op.apply(x11)
    d, idd = op.solve(r, mg, 1e-11, 800)
    assert idd.flag in (0, 3) and idd.relres <= 1e-10, (idd.flag, idd.relres)
    x11 = x11 + d
    if blk.n <= 60000:
        Ah = V.field_csr(np.ones((ne[2], ne[1], ne[0])) if f is None else f, blk.h)
        xr = sla.spsolve(Ah.tocsc(), b.cpu().numpy())
        assert np.linalg.norm(x11.cpu().numpy() - xr) <= 1e-9 * np.linalg.norm(xr)
    else:
        xj, ij = op.solve(b, op.jacobi(), 1e-13, 100000)
        assert ij.flag in (0, 3)
        assert float((x11 - xj).norm()) <= 1e-9 * float(xj.norm()), float((x11 - xj).norm() / xj.norm())


def test_launches_per_iteration(cuda):
    """Launches per MG-PCG iteration depend on the level count only: 25^3 under "any" (5 levels) equals 32^3 under the
    default (5 levels), and "any" on 32^3 equals the default there."""
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid

    def per_iter(op, M, b):
        ls = []
        for maxiter in (6, 12):
            _, info = op.solve(b, M, 1e-30, maxiter, fixed_iters=True, check_every=6)
            ls.append(info.launches)
        return ls[1] - ls[0]

    blk, op, mg = _setup(cuda, (25, 25, 25))
    blk32, op32, mg32 = _setup(cuda, (32, 32, 32))
    ev32 = HexMultigrid(op32, blk32)
    assert len(mg.level_shapes()) == len(ev32.level_shapes()) == 5
    b, b32 = load_vector(blk, device=cuda), load_vector(blk32, device=cuda)
    p = per_iter(op, mg, b)
    assert p == per_iter(op32, ev32, b32) == per_iter(op32, mg32, b32), p


def test_refusals_leak_nothing(cuda):
    import gc
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    blk, op, mg = _setup(cuda, (5, 4, 3))
    for bad in (-1, len(mg.level_shapes())):
        with pytest.raises(_lib.PcgbError):
            _lib.check(_lib.load().pcgb_mg_level_box(mg.handle, bad, (ctypes.c_int32 * 3)()), "pcgb_mg_level_box")
    del mg
    gc.collect()

    def refused(exc, fn, *a, **kw):
        torch.cuda.synchronize()
        free0, _ = torch.cuda.mem_get_info(cuda)
        with pytest.raises(exc):
            fn(*a, **kw)
        gc.collect()
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info(cuda)[0] >= free0

    for ne in ((2, 2, 2), (1, 2, 1), (2, 1, 2)):       # nothing to coarsen
        b2 = HexBlock(ne, (0, 0, 0), ne, h=0.5)
        refused(_lib.PcgbError, HexMultigrid, SubdomainOperator(generate_matrix(b2, cuda)), b2, coarsening="any")
    part = HexBlock((10, 4, 3), (5, 0, 0), (5, 4, 3), h=0.1)    # e0 != 0: not the whole mesh
    refused(_lib.PcgbError, HexMultigrid, SubdomainOperator(generate_matrix(part, cuda)), part, coarsening="any")
    refused(ValueError, HexMultigrid, op, blk, coarsening="odd")
    refused(ValueError, HexMultigrid, op, blk, coarsening="any", E_field=np.ones((3, 4, 4)))
    f = np.ones((3, 4, 5))
    f[1, 2, 3] = -1.0
    refused(_lib.PcgbError, HexMultigrid, op, blk, coarsening="any", E_field=f)
    comm = Communicator(0, 1, None, device=cuda)
    refused(_lib.PcgbError, HexMultigrid, SubdomainOperator(op.A, comm=comm), blk, coarsening="any")

    class TwoRanks:      # what HexMultigrid sees of a multi-rank operator before anything else
        comm = type("C", (), {"nranks": 2, "rank": 0})()
        n, device = op.n, op.device
    refused(ValueError, HexMultigrid, TwoRanks(), blk, coarsening="any")
    refused(ValueError, HexMultigrid, TwoRanks(), blk, coarsening="any", E_field=np.ones((3, 4, 5)))
