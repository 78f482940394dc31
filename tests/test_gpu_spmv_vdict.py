"""The value dictionary of the node-block SpMV (spmv.cuh build_vdict / k_spmv_bsr3<VD>): when a matrix has at most 1024
bitwise-distinct 3x3 blocks the kernel streams a 16-bit id per block and reads the values from a shared-memory copy.

The products must be the same bits as the kernel that streams the values (PCGB_SPMV_VDICT=0): y, the fused x.y of the
split launch, and whole PCG / MG-PCG solves.  The dictionary is keyed by bit pattern, so blocks that differ only in the sign
of a zero or a NaN payload are distinct; a matrix with more distinct blocks than the dictionary holds keeps today's plan."""
import os

import numpy as np
import pytest

from tests import spmv_cases as C

pytestmark = pytest.mark.gpu
DMAX = 1024
_GATE = {"PCGB_BSR_MIN_UNIFORM_PCT": "0"}   # small matrices are mostly boundary: keep the regularity gate out of it


def _env(monkeypatch, env):
    for k in list(os.environ):
        if k.startswith("PCGB_SPMV_") or k.startswith("PCGB_BSR_"):
            monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def _bits(t):
    import torch
    return t.contiguous().view(torch.int64)


def _products(monkeypatch, rp, col, val, shape, env, x, boundary):
    """(vd, plan_info, y, y of the split launch, x.y of the split launch) of a plan built under `env`."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    _env(monkeypatch, env)
    M = CsrMatrix(rp, col, val, shape)
    vd, info = M.value_dict_blocks(), M.plan_info()
    y = torch.full((shape[0],), float("nan"), dtype=torch.float64, device=val.device)
    M.spmv(x, out=y)
    M.set_boundary_rows(boundary)
    ys = torch.full_like(y, float("nan"))
    _, d = M.spmv_split(x, with_dot=True, out=ys)
    torch.cuda.synchronize()
    del M
    return vd, info, y, ys, d


def _assert_same_bits(monkeypatch, rp, col, val, shape, env, seed=0):
    """Plan under env (+ dictionary switch on / off): returns (vd, info on, info off); asserts bit-identical products."""
    import torch
    dev = val.device
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(shape[1], dtype=torch.float64, device=dev, generator=g)
    n = shape[0]
    boundary = torch.unique(torch.randint(0, max(n, 1), (max(n // 50, 1),), device=dev, generator=g)).to(torch.int32)
    vd, info, y, ys, d = _products(monkeypatch, rp, col, val, shape, env, x, boundary)
    vd0, info0, y0, ys0, d0 = _products(monkeypatch, rp, col, val, shape, dict(env, PCGB_SPMV_VDICT="0"), x, boundary)
    assert vd0 == 0
    assert torch.equal(_bits(y), _bits(y0)), "y differs from the kernel that streams the values"
    assert torch.equal(_bits(ys), _bits(ys0)) and torch.equal(_bits(ys), _bits(y)), "split launch differs"
    assert torch.equal(_bits(d), _bits(d0)), ("fused x.y differs", float(d), float(d0))
    return vd, info, info0, (x, y)


def _tensors(A, dev, index64=False):
    import torch
    rp = torch.from_numpy(A.indptr.astype(np.int64 if index64 else np.int32)).to(dev)
    return rp, torch.from_numpy(A.indices.astype(np.int32)).to(dev), torch.from_numpy(A.data.copy()).to(dev)


def _block_positions(A):
    """(blocks, 9) positions in A.data of the 9 values of every 3x3 block, in block order (node, then column)."""
    ip = A.indptr.astype(np.int64)
    a0 = ip[0:-1:3]
    L = ip[1::3] - a0
    nb = L // 3
    node = np.repeat(np.arange(nb.size), nb)
    t = np.arange(node.size) - np.repeat(np.cumsum(nb) - nb, nb)
    base = a0[node] + 3 * t
    r, c = np.repeat(np.arange(3), 3), np.tile(np.arange(3), 3)     # row-major entries of the block
    return base[:, None] + r[None, :] * L[node][:, None] + c[None, :]


def _with_dictionary(A, nd, seed):
    """A copy of the node-block matrix A whose blocks take exactly nd distinct values, repeated at random positions."""
    rng = np.random.default_rng(seed)
    pos = _block_positions(A)
    assert pos.shape[0] >= nd
    ids = rng.integers(0, nd, pos.shape[0])
    ids[rng.choice(pos.shape[0], nd, replace=False)] = np.arange(nd)   # every value occurs
    dic = rng.standard_normal((nd, 9))
    B = A.copy()
    B.data = np.empty_like(A.data)
    B.data[pos] = dic[ids]
    return B


# ------------------------------------------------------------------------------------------------ hex boxes
HEX = [  # (ng, e0, ne, mode): e0 != 0 boxes have no clamped face; mode 1 = the default size rule, 2 = forced
    ((12, 10, 8), (0, 0, 0), (12, 10, 8), "2"),
    ((40, 40, 40), (4, 2, 3), (20, 16, 12), "2"),
    ((40, 40, 40), (0, 5, 7), (9, 17, 6), "2"),
    ((64, 64, 64), (1, 0, 0), (3, 5, 4), "2"),
    ((32, 32, 32), (0, 0, 0), (32, 32, 32), "1"),
    ((96, 96, 96), (20, 30, 10), (40, 36, 28), "1"),
]


@pytest.mark.parametrize("ng,e0,ne,mode", HEX)
def test_hex_dictionary_is_chosen_and_bit_identical(cuda, monkeypatch, ng, e0, ne, mode):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    blk = HexBlock(ng, e0, ne, h=1.0 / ng[0])
    A = generate_matrix(blk, device=cuda)
    env = dict(_GATE, PCGB_SPMV_VDICT=mode)
    vd, info, info0, _ = _assert_same_bits(monkeypatch, A.rowptr, A.col, A.val, A.shape, env)
    assert 1 <= vd <= 729, vd                  # 27 neighbour offsets x 27 face classes
    assert info["index_mode"] == 2 and info["staged"] == 2 and info0["index_mode"] == 2 and info0["staged"] == 2


def test_default_plan_on_a_hex_box(cuda, monkeypatch):
    """Without any switch a 48^3 box takes the dictionary, and the plan fields the bench reads are unchanged."""
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    _env(monkeypatch, {})
    A = generate_matrix(HexBlock((48,) * 3, (0, 0, 0), (48,) * 3, h=1.0 / 48), device=cuda)
    assert 1 <= A.value_dict_blocks() <= 729
    info = A.plan_info()
    assert info["staged"] == 2 and info["index_mode"] == 2 and info["split_rows"] == 0
    assert A.stream_bytes() < 0.3 * A.spmv_bytes()      # ids + indices instead of 8 B per non-zero
    _env(monkeypatch, {"PCGB_SPMV_VDICT": "0"})
    M = CsrMatrix(A.rowptr, A.col, A.val, A.shape)
    assert M.value_dict_blocks() == 0 and M.stream_bytes() > 5 * A.stream_bytes()


# ------------------------------------------------------------------------------------------------ synthetic blocks
@pytest.mark.parametrize("nd", [1, DMAX - 1, DMAX, DMAX + 1])
def test_dictionary_limit(cuda, monkeypatch, nd):
    A = _with_dictionary(C.nb_many(), nd, seed=nd)
    rp, col, val = _tensors(A, cuda)
    env = dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="600")
    vd, info, info0, _ = _assert_same_bits(monkeypatch, rp, col, val, A.shape, env, seed=nd)
    if nd <= DMAX:
        assert vd == nd
        assert info["index_mode"] == 2 and info["staged"] == 2
    else:
        assert vd == 0 and info == info0      # no dictionary: exactly the plan without one


@pytest.mark.parametrize("case", ["nb-empty", "nb-many", "nb-mixed", "nb-singleton", "nb-rect", "nb-1-node", "nb-2-nodes"])
@pytest.mark.parametrize("tile", [None, 300, 600])
def test_repeats_across_tiles_stages_and_empty_nodes(cuda, monkeypatch, case, tile):
    """Few distinct blocks repeated at random over many small tiles (every ring stage wraps), empty nodes and runs of
    them, single-block nodes, rectangular matrices and matrices smaller than one tile; checked entrywise as well."""
    build = {"nb-empty": lambda: C.nb_empty()[0], "nb-many": C.nb_many, "nb-mixed": C.nb_mixed, "nb-singleton": C.nb_singleton,
             "nb-rect": C.nb_rect, "nb-1-node": lambda: C.nb_small(1), "nb-2-nodes": lambda: C.nb_small(2)}[case]
    A0 = build().tocsr()
    nd = min(37, A0.nnz // 9)
    A = _with_dictionary(A0, nd, seed=len(case))
    rp, col, val = _tensors(A, cuda)
    env = dict(_GATE, PCGB_SPMV_VDICT="2")
    if tile:
        env["PCGB_SPMV_TILE"] = str(tile)
    vd, info, _, (x, y) = _assert_same_bits(monkeypatch, rp, col, val, A.shape, env)
    assert vd == nd and info["index_mode"] == 2
    if tile == 300 and case == "nb-many":
        assert info["ntiles"] >= 6 * info["resident_ctas"], info
    y_ref, scale = C.ref_spmv(A, x.cpu().numpy())
    err = np.abs(y.cpu().numpy().astype(np.longdouble) - y_ref) / (scale + 1e-300)
    assert float(err.max(initial=0.0)) <= 1e-13


def test_signed_zero_and_nan_payloads_are_distinct(cuda, monkeypatch):
    A = C.nb_many(nn=3001).tocsr()
    pos = _block_positions(A)
    base = np.arange(1.0, 10.0)
    base[1] = 0.0
    variants = np.tile(base, (4, 1))
    variants[1, 1] = -0.0                                                    # sign of a zero
    variants[2, 5] = np.array([0x7FF8000000000001], dtype=np.uint64).view(np.float64)[0]   # two NaN payloads
    variants[3, 5] = np.array([0x7FF8000000000002], dtype=np.uint64).view(np.float64)[0]
    ids = np.zeros(pos.shape[0], dtype=np.int64)
    ids[100:200] = 1
    ids[1000] = 2
    ids[2000] = 3
    B = A.copy()
    B.data = np.empty_like(A.data)
    B.data[pos] = variants[ids]
    rp, col, val = _tensors(B, cuda)
    vd, *_ = _assert_same_bits(monkeypatch, rp, col, val, B.shape, dict(_GATE, PCGB_SPMV_VDICT="2"))
    assert vd == 4
    # the same matrix with the variants collapsed has one block
    B.data[pos] = variants[np.zeros_like(ids)]
    rp, col, val = _tensors(B, cuda)
    vd, *_ = _assert_same_bits(monkeypatch, rp, col, val, B.shape, dict(_GATE, PCGB_SPMV_VDICT="2"))
    assert vd == 1


def test_int64_offsets(cuda, monkeypatch):
    A = _with_dictionary(C.nb_empty()[0].tocsr(), 50, seed=3)
    rp, col, val = _tensors(A, cuda, index64=True)
    vd, info, *_ = _assert_same_bits(monkeypatch, rp, col, val, A.shape, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="600"))
    assert vd == 50 and info["index_mode"] == 2


# ------------------------------------------------------------------------------------------------ full size
def test_256_box_past_2_31_offsets(cuda, monkeypatch):
    """256^3 (64-bit row offsets, 4.5e8 blocks): dictionary chosen, y bit-identical, rows around offset 2^31 included."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 70e9:
        pytest.skip("needs ~70 GB of free device memory")
    _env(monkeypatch, {})
    B = 256
    A = generate_matrix(HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B), device=cuda)
    assert A.rowptr.dtype == torch.int64 and 1 <= A.value_dict_blocks() <= 729
    x = torch.randn(A.shape[1], dtype=torch.float64, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5))
    y = A.spmv(x).clone()
    r31 = int(torch.searchsorted(A.rowptr, torch.tensor([2**31], dtype=torch.int64, device=cuda)).item())
    rows = torch.arange(max(r31 - 600, 0), min(r31 + 600, A.shape[0]), device=cuda)
    from pcg_mpi_solver_b200.csr import CsrMatrix
    _env(monkeypatch, {"PCGB_SPMV_VDICT": "0"})
    M = CsrMatrix(A.rowptr, A.col, A.val, A.shape)
    assert M.value_dict_blocks() == 0
    y0 = M.spmv(x)
    assert torch.equal(_bits(y[rows]), _bits(y0[rows])) and bool(torch.isfinite(y[rows]).all())
    assert torch.equal(_bits(y), _bits(y0))


@pytest.fixture(scope="module")
def box128(cuda):
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, load_vector
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 24e9:
        pytest.skip("needs ~20 GB of free device memory")
    blk = HexBlock((128,) * 3, (0, 0, 0), (128,) * 3, h=1.0 / 128)
    A = generate_matrix(blk, device=cuda)
    return blk, A, load_vector(blk, device=cuda)


def _solve(monkeypatch, box, env, mg):
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk, A, b = box
    _env(monkeypatch, env)
    M = CsrMatrix(A.rowptr, A.col, A.val, A.shape)
    op = SubdomainOperator(M)
    pre = HexMultigrid(op, blk) if mg else op.jacobi()
    x, info = op.solve(b, pre, 0.0, 12 if mg else 40, fixed_iters=True, record_resvec=True, trace=True, check_every=5)
    return M.value_dict_blocks(), x, info


@pytest.mark.parametrize("mg", [False, True])
def test_pcg_128_bit_identical(box128, monkeypatch, mg):
    import torch
    vd, x, info = _solve(monkeypatch, box128, {}, mg)
    vd0, x0, info0 = _solve(monkeypatch, box128, {"PCGB_SPMV_VDICT": "0"}, mg)
    assert 1 <= vd <= 729 and vd0 == 0
    assert torch.equal(_bits(x), _bits(x0))
    assert np.array_equal(info.resvec.view(np.int64), info0.resvec.view(np.int64))
    assert info.trace.tobytes() == info0.trace.tobytes() and info.iters == info0.iters


def test_concrete_refuses_the_dictionary(cuda, monkeypatch):
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "concrete.zip")
    if not os.path.exists(p):
        pytest.skip("data/concrete.zip not staged (oracle/stage_ref.py)")
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.partition import assemble_csr_device, partition_mesh
    sub = partition_mesh(p, 1, assemble=False)[0]
    rp, col, val = assemble_csr_device(sub, cuda)
    for env in ({}, dict(_GATE, PCGB_SPMV_VDICT="2")):   # default plan, and the node-block gate opened with the forced mode
        _env(monkeypatch, env)
        M = CsrMatrix(rp, col, val, (sub.n, sub.n))
        assert M.value_dict_blocks() == 0, env
        del M
