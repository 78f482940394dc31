"""Voxel models on the device (pcgb_hex_fill_field, pcgb_mg_create_field, hexmesh E_field, HexMultigrid(E_field=...)):
the field CSR entrywise against a long-double assembly, the EBE operators and the METIS/device-assembly pipeline with the
field, Jacobi-PCG against the oracle, every Galerkin coarse level against scipy P^T A P, the V-cycle's parts against the
host restatement (tests/voxel_cases.py), MG-PCG across the contrast range, launch counts and refusals."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import gmg_cases as G
from tests import voxel_cases as V

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -53


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _csr_host(A):
    rp = A.rowptr.cpu().numpy().astype(np.int64)
    return sp.csr_matrix((A.val.cpu().numpy(), A.col.cpu().numpy(), rp), shape=A.shape)


def _setup(cuda, field, kind="csr", degree=2, lo=0.25):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = tuple(int(v) for v in reversed(field.shape))
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0])
    A = generate_matrix(blk, device=cuda, E_field=field) if kind == "csr" else \
        generate_ebe(blk, device=cuda, ordered=kind == "ebe_ordered", E_field=field)
    op = SubdomainOperator(A)
    return blk, op, HexMultigrid(op, blk, degree=degree, lo=lo, E_field=field)


@pytest.mark.parametrize("ng,e0,ne", [((8, 6, 4), (0, 0, 0), (8, 6, 4)), ((8, 6, 4), (4, 0, 0), (4, 6, 4)),
                                      ((12, 10, 8), (3, 2, 1), (5, 4, 6)), ((40, 36, 34), (0, 0, 0), (40, 36, 34))])
def test_field_csr_entrywise_and_reproducible(cuda, ng, e0, ne):
    """rowptr and col identical to the uniform generator's; every value within (k+2) 2^-53 sum|terms| of a long-double sum of
    the same k element terms; a repeat is bit-identical.  Boxes with and without the clamped face, e0 != 0, and a larger
    non-cubic box (51 800 free nodes)."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, block_field, generate_matrix, hex_element_stiffness
    blk = HexBlock(ng, e0, ne, h=0.5)
    f = block_field(V.random_field(ng, seed=sum(ne)), blk)
    A = generate_matrix(blk, device=cuda, E_field=f)
    U = generate_matrix(blk, device=cuda)
    assert torch.equal(A.rowptr, U.rowptr) and torch.equal(A.col, U.col)
    rows, cols, ref, mag, k = V.assemble_ld(V.fine_elements(f, blk.h, hex_element_stiffness(1.0, blk.nu)), e0)
    H = _csr_host(A).tocoo()
    assert np.array_equal(H.row, rows) and np.array_equal(H.col, cols)
    err = np.abs(H.data.astype(np.longdouble) - ref)
    assert np.all(err <= (k + 2) * EPS * mag), float(np.max(err / mag))
    B = generate_matrix(blk, device=cuda, E_field=torch.from_numpy(f).to(cuda))
    assert torch.equal(A.val, B.val)


def test_block256_field_int64_offsets(cuda):
    """The 256^3 voxel box (4.08e9 non-zeros, int64 row offsets): rows around the offsets 2^31 and 3 * 2^30, and the first and
    last rows, against a long-double sum of Ck_e Ke over the same elements; rowptr and the sampled columns equal to the
    uniform generator's (generated after the field matrix is freed: both do not fit at once)."""
    import gc
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, hex_element_stiffness
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 60e9:
        pytest.skip("needs ~60 GB of free device memory")
    ng = (256, 256, 256)
    blk = HexBlock(ng, (0, 0, 0), ng, h=1.0 / 256)
    f = V.random_field(ng, seed=256)
    A = generate_matrix(blk, device=cuda, E_field=f)
    n, nnz = A.shape[0], A.nnz
    assert A.rowptr.dtype == torch.int64 and 2**31 < nnz < 2**32
    cross = torch.searchsorted(A.rowptr, torch.tensor([2**31, 3 * 2**30], dtype=torch.int64, device=cuda), right=True) - 1
    assert int(A.rowptr[cross[0]]) <= 2**31 < int(A.rowptr[cross[0] + 1])
    half = 1500
    wins = [(0, half), (n - half, n)] + [(max(0, r - half), min(n, r + half)) for r in cross.tolist()]
    rowptr = A.rowptr.clone()
    got = []
    for a, e in wins:
        rp = A.rowptr[a:e + 1].cpu().numpy()
        k0, k1 = int(rp[0]), int(rp[-1])
        got.append((a, e, rp, A.col[k0:k1].cpu().numpy(), A.val[k0:k1].cpu().numpy()))
    del A
    gc.collect()
    torch.cuda.empty_cache()
    ke = hex_element_stiffness(1.0, blk.nu)
    for a, e, rp, col, val in got:
        rows = np.repeat(np.arange(a, e), np.diff(rp))
        ref, mag, k = V.field_entries_ld(f, blk.h, ke, rows, col)
        assert np.all(k >= 1)
        err = np.abs(val.astype(np.longdouble) - ref)
        assert np.all(err <= (k + 2) * EPS * mag), (a, e, float(np.max(err / mag)))
    U = generate_matrix(blk, device=cuda)
    assert torch.equal(U.rowptr, rowptr)
    for a, e, rp, col, _ in got:
        assert np.array_equal(U.col[int(rp[0]):int(rp[-1])].cpu().numpy(), col), (a, e)
    del U, rowptr
    gc.collect()
    torch.cuda.empty_cache()


def test_field_tensor_devices(cuda):
    """A field tensor on the CPU or on the operator's device is taken whatever spelling names that device ('cuda',
    'cuda:0'), by the CSR generator and by both EBE operators; the three give the same products."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix
    ng = (6, 4, 4)
    blk = HexBlock(ng, (0, 0, 0), ng, h=0.25)
    f = V.random_field(ng, seed=13)
    x = _t(np.random.default_rng(4).standard_normal(blk.n), cuda)
    ref = generate_matrix(blk, device=cuda, E_field=f).spmv(x)
    for t in (torch.from_numpy(f), torch.from_numpy(f).to(cuda)):
        for dev in ("cuda", cuda):
            assert torch.equal(generate_matrix(blk, device=dev, E_field=t).spmv(x), ref)
            for ordered in (False, True):
                y = generate_ebe(blk, device=dev, ordered=ordered, E_field=t).apply_local(x)
                assert float((y - ref).abs().max()) <= 1e-13 * float(ref.abs().max())


def test_device_assembly_of_the_field_model(cuda):
    """partition_mesh(hex_mdf_model(E_field), 1) assembled on the device is the generator's matrix within the same bound."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, hex_element_stiffness, hex_mdf_model
    from pcg_mpi_solver_b200.partition import assemble_csr_device, partition_mesh
    ng, h = (6, 5, 4), 1.0 / 6
    f = V.random_field(ng, seed=5)
    sub = partition_mesh(hex_mdf_model(ng, h=h, E_field=f), 1, assemble=False)[0]
    rp, col, val = assemble_csr_device(sub, cuda)
    D = sp.csr_matrix((val.cpu().numpy(), col.cpu().numpy(), rp.cpu().numpy().astype(np.int64)), shape=(sub.n, sub.n))
    # the part's free dofs -> the generator's free numbering (x fastest, global x = 0 dropped)
    g = sub.dof_eff_global
    node, d = g // 3, g % 3
    gx, gy, gz = node % (ng[0] + 1), (node // (ng[0] + 1)) % (ng[1] + 1), node // ((ng[0] + 1) * (ng[1] + 1))
    perm = 3 * ((gz * (ng[1] + 1) + gy) * ng[0] + gx - 1) + d
    P = sp.csr_matrix((np.ones(sub.n), (perm, np.arange(sub.n))), shape=(sub.n, sub.n))
    D = (P @ D @ P.T).tocsr()
    blk = HexBlock(ng, (0, 0, 0), ng, h=h)
    A = _csr_host(generate_matrix(blk, device=cuda, E_field=f))
    _, _, _, mag, k = V.assemble_ld(V.fine_elements(f, h, hex_element_stiffness(1.0, blk.nu)))
    diff = (D - A).tocoo()
    Mag = sp.csr_matrix((mag.astype(np.float64) * (k + 2) * 2 * EPS, (A.tocoo().row, A.tocoo().col)), shape=A.shape)
    assert np.all(np.abs(diff.data) <= np.asarray(Mag[diff.row, diff.col]).ravel())
    assert D.nnz == A.nnz


@pytest.mark.parametrize("ordered", [False, True])
def test_ebe_with_field_matches_csr(cuda, ordered):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, block_field, generate_ebe, generate_matrix
    ng = (10, 8, 6)
    f = V.random_field(ng, seed=9, lo=1.0, hi=1000.0)
    for e0, ne in (((0, 0, 0), ng), ((4, 2, 0), (6, 6, 6))):
        blk = HexBlock(ng, e0, ne, h=0.25)
        fb = block_field(f, blk)
        A = generate_matrix(blk, device=cuda, E_field=fb)
        E = generate_ebe(blk, device=cuda, ordered=ordered, E_field=fb)
        x = np.random.default_rng(2).standard_normal(blk.n)
        y = E.apply_local(_t(x, cuda)).cpu().numpy()
        H = _csr_host(A)
        assert np.all(np.abs(y - H @ x) <= 1e-13 * (abs(H) @ np.abs(x))), (ordered, e0)


def test_jacobi_pcg_matches_oracle(cuda):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ng = (8, 6, 6)
    f = V.two_phase(ng, 10.0, seed=2)
    blk = HexBlock(ng, (0, 0, 0), ng, h=1.0 / 8)
    A = generate_matrix(blk, device=cuda, E_field=f)
    b = load_vector(blk, device=cuda)
    op = SubdomainOperator(A)
    x, info = op.solve(b, op.jacobi(), 1e-13, 5000)
    flag, iters = info.flag, info.iters
    As = V.field_csr(f, blk.h)
    ref = R.ref_pcg([R.CsrPart(As, b.cpu().numpy())], [1.0 / As.diagonal()], 1e-13, 5000)
    assert flag == ref["Flag"] and abs(iters - ref["Iter"]) <= 2, (flag, iters, ref["Flag"], ref["Iter"])
    xr = ref["X"][0]
    assert np.linalg.norm(x.cpu().numpy() - xr) <= 1e-10 * np.linalg.norm(xr)


@pytest.mark.parametrize("ne", [(16, 16, 16), (16, 8, 12), (24, 16, 8)])
def test_level_matrices_equal_ptap(cuda, ne):
    """Every smoothed coarse level: the uniform generator's pattern, values equal to scipy P^T A P of the level below (from
    the host fine matrix) within 1e-12 of the row's largest entry.  Level 0 and the coarsest are refused."""
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    f = V.random_field(ne, seed=11, lo=1.0, hi=100.0)
    blk, op, mg = _setup(cuda, f)
    uni = HexMultigrid(op, blk)
    info = mg.info()
    assert info["levels"] >= 3 and info["n"] == uni.info()["n"]
    A = V.field_csr(f, blk.h)
    lv = G.levels_of(ne)
    for l in range(1, info["levels"] - 1):
        A = (G.prolongation_matrix(lv[l - 1]).T @ A @ G.prolongation_matrix(lv[l - 1])).tocsr()
        rp, col, val = mg.level_matrix(l)
        urp, ucol, _ = uni.level_matrix(l)
        assert torch.equal(rp, urp) and torch.equal(col, ucol)
        D = sp.csr_matrix((val.cpu().numpy(), col.cpu().numpy(), rp.cpu().numpy()), shape=A.shape)
        assert (D != D.T).nnz == 0          # mirrored element matrices: exactly symmetric
        diff = abs(D - A).max(axis=1).toarray().ravel()
        rowmax = abs(A).max(axis=1).toarray().ravel()
        assert np.all(diff <= 1e-12 * rowmax), (l, float(np.max(diff / rowmax)))
    for bad in (0, info["levels"] - 1, -1):
        with pytest.raises(_lib.PcgbError, match=r"\(-1\)"):
            mg.level_matrix(bad)
    # the coarsest level, built from the Galerkin element matrices of the level above it (fnx != fny on the non-cubic
    # boxes), against a dense solve of the host Galerkin coarsest matrix
    Ac = V.level_matrices(f, blk.h)[-1].toarray()
    r = np.random.default_rng(12).standard_normal(Ac.shape[0])
    z = mg.coarse_solve(_t(r, cuda)).cpu().numpy()
    zr = G.refined_solve(Ac, r)
    assert np.linalg.norm(z - zr) <= 1e-10 * np.linalg.norm(zr)


def test_setup_is_bit_identical(cuda):
    import torch
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    f = V.two_phase((16, 16, 16), 100.0, seed=4)
    blk, op, mg = _setup(cuda, f)
    mg2 = HexMultigrid(op, blk, E_field=f)
    for l in range(1, mg.info()["levels"] - 1):
        assert all(torch.equal(a, b) for a, b in zip(mg.level_matrix(l), mg2.level_matrix(l)))
    r = _t(np.random.default_rng(1).standard_normal(mg.n), cuda)
    assert torch.equal(mg.apply(r), mg2.apply(r))
    assert mg.info()["lambda"] == mg2.info()["lambda"]
    s = mg.setup_info()
    assert s["galerkin_ms"] > 0 and s["element_matrix_peak_bytes"] == 4608 * (8 ** 3 + 4 ** 3)


@pytest.mark.parametrize("kind", ["csr", "ebe_ordered", "ebe"])
@pytest.mark.parametrize("degree", [1, 2, 3])
def test_vcycle_parts_match_host(cuda, kind, degree):
    """lambda per level against the host Lanczos on the host Galerkin levels (1e-10); fed the device's lambda and D^-1:
    one smoothing per level (1e-12), the whole V-cycle (1e-12), its symmetry (1e-12) and the coarse solve against a
    dense solve of the Galerkin coarsest matrix."""
    ne = (16, 16, 16)
    f = V.two_phase(ne, 100.0, seed=6)
    blk, op, mg = _setup(cuda, f, kind, degree=degree)
    info = mg.info()
    H0 = V.HostFieldMultigrid(f, blk.h, degree=degree)
    lam = info["lambda"][:info["levels"] - 1]
    assert np.allclose(lam, H0.lam, rtol=1e-10, atol=0), (lam, H0.lam)
    H = V.HostFieldMultigrid(f, blk.h, degree=degree, lambdas=lam, minv=op.jacobi().cpu().numpy(), mats=H0.mats)
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
    Ac = H0.mats[-1].toarray()
    r = rng.standard_normal(Ac.shape[0])
    z = mg.coarse_solve(_t(r, cuda)).cpu().numpy()
    zr = G.refined_solve(Ac, r)
    assert np.linalg.norm(z - zr) <= 1e-10 * np.linalg.norm(zr)


def test_constant_field_matches_uniform_hierarchy(cuda):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    ne = (16, 16, 16)
    f = np.full(ne, 3.5)
    blk, op, mg = _setup(cuda, f)
    blk.E = 3.5
    uni = HexMultigrid(op, blk)
    u = np.random.default_rng(8).standard_normal(mg.n)
    a, b = mg.apply(_t(u, cuda)).cpu().numpy(), uni.apply(_t(u, cuda)).cpu().numpy()
    assert np.linalg.norm(a - b) <= 1e-12 * np.linalg.norm(b)


@pytest.mark.parametrize("m", [24, 32, 64])
@pytest.mark.parametrize("contrast", [1.0, 10.0, 100.0, 1000.0])
def test_mg_pcg_across_contrast(cuda, m, contrast):
    """MG-PCG reaches flag 0 at 1e-8; x at 1e-11 against a sparse direct solve (24^3) or long-tolerance Jacobi-PCG.  At high
    contrast the 1e-11 solve may stagnate (flag 3) just above its tolerance; its relres must still be below 1e-10."""
    import scipy.sparse.linalg as sla
    from pcg_mpi_solver_b200.hexmesh import load_vector
    f = V.two_phase((m, m, m), contrast, seed=m, radii=(1.0, m / 8))
    blk, op, mg = _setup(cuda, f)
    b = load_vector(blk, device=cuda)
    x, info = op.solve(b, mg, 1e-8, 300)
    assert info.flag == 0, (info.flag, info.iters)
    x11, info11 = op.solve(b, mg, 1e-11, 400)
    assert info11.flag in (0, 3) and info11.relres <= 1e-10, (info11.flag, info11.relres)
    if m == 24:
        xr = sla.spsolve(V.field_csr(f, blk.h).tocsc(), b.cpu().numpy())
        assert np.linalg.norm(x11.cpu().numpy() - xr) <= 1e-8 * np.linalg.norm(xr)
    else:
        xj, ij = op.solve(b, op.jacobi(), 1e-11, 60000)
        assert ij.flag in (0, 3)
        assert float((x11 - xj).norm()) <= 1e-6 * float(xj.norm()), float((x11 - xj).norm() / xj.norm())


def test_launches_per_iteration_match_uniform_handle(cuda):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    f = V.two_phase((16, 16, 16), 10.0, seed=1)
    blk, op, mg = _setup(cuda, f)
    uni = HexMultigrid(op, blk)
    b = load_vector(blk, device=cuda)
    per = []
    for M in (mg, uni):
        ls = []
        for maxiter in (6, 12):
            _, info = op.solve(b, M, 1e-30, maxiter, fixed_iters=True, check_every=6)
            ls.append(info.launches)
        per.append(ls[1] - ls[0])
    assert per[0] == per[1], per


def test_refusals_leak_nothing(cuda):
    import gc
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    ne = (8, 8, 8)
    f = V.random_field(ne, seed=1)
    blk, op, mg = _setup(cuda, f)
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

    for bad in (f[:, :, :-1], f.astype(np.float32), torch.from_numpy(f).to("meta"), f.tolist()):
        refused(ValueError, HexMultigrid, op, blk, E_field=bad)
        refused(ValueError, generate_matrix, blk, cuda, bad)
    for v in (0.0, -1.0, float("nan"), float("inf")):
        g = f.copy()
        g[3, 2, 1] = v
        refused(_lib.PcgbError, HexMultigrid, op, blk, E_field=g)
        refused(_lib.PcgbError, generate_matrix, blk, cuda, g)
    odd = HexBlock((8, 8, 5), (0, 0, 0), (8, 8, 5), h=1 / 8)     # a box that does not coarsen
    fo = np.ones((5, 8, 8))
    refused(_lib.PcgbError, HexMultigrid, SubdomainOperator(generate_matrix(odd, cuda, fo)), odd, E_field=fo)
    comm = Communicator(0, 1, None, device=cuda)
    refused(_lib.PcgbError, HexMultigrid, SubdomainOperator(op.A, comm=comm), blk, E_field=f)

    class TwoRanks:      # what HexMultigrid sees of a multi-rank operator before anything else
        comm = type("C", (), {"nranks": 2, "rank": 0})()
        n, device = op.n, op.device
    refused(ValueError, HexMultigrid, TwoRanks(), blk, E_field=f)
