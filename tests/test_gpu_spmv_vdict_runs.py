"""The run-compressed index stream of the dictionary node-block SpMV (spmv.cuh k_vd_runs / k_spmv_bsr3_vd).

Within a tile, a node whose blocks are its predecessor's shifted by one node (staged x position + 3, same dictionary id,
same block count) joins its run, and the kernel reads the run head's block words for it.  The products must stay the same
bits as the kernel that streams the values (PCGB_SPMV_VDICT=0), and the share of nodes in runs must be what a host
restatement of the rule gives on the plan's own tiles: runs end at tile boundaries, and a tile with more than 8 segments
is stored explicitly."""
import numpy as np
import pytest

from tests import spmv_cases as C
from tests.nodeblock_cases import expected_run_nodes
from tests.test_gpu_spmv_vdict import _GATE, _assert_same_bits, _bits, _block_positions, _env, _tensors, _with_dictionary

pytestmark = pytest.mark.gpu


def _run_share(M):
    return M.value_dict_run_share()


def _check(monkeypatch, A, env, expect_runs=None, seed=0, index64=False):
    """Bit identity with PCGB_SPMV_VDICT=0, the long-double bound, and the run share against the host restatement."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    rp, col, val = _tensors(A, "cuda", index64=index64)
    vd, info, _, (x, y) = _assert_same_bits(monkeypatch, rp, col, val, A.shape, env, seed=seed)
    assert vd >= 1 and info["index_mode"] == 2, (vd, info)
    y_ref, scale = C.ref_spmv(A, x.cpu().numpy())
    err = np.abs(y.cpu().numpy().astype(np.longdouble) - y_ref) / (scale + 1e-300)
    assert float(err.max(initial=0.0)) <= 1e-13
    _env(monkeypatch, env)
    M = CsrMatrix(rp, col, val, A.shape)
    share = _run_share(M)
    nn = A.shape[0] // 3
    want = expected_run_nodes(A, M.plan_info()["tile_items"])
    assert share == want / nn, (share * nn, want)
    if expect_runs is not None:
        assert (want > 0) == expect_runs, want
    del M
    torch.cuda.synchronize()
    return want, info


# ------------------------------------------------------------------------------------------------ hex boxes
HEX = [  # (ng, e0, ne): e0 != 0 boxes have no clamped face; x-rows shorter and longer than a tile (~24 nodes)
    ((12, 10, 8), (0, 0, 0), (12, 10, 8)),
    ((40, 40, 40), (4, 2, 3), (20, 16, 12)),
    ((40, 40, 40), (0, 5, 7), (9, 17, 6)),
    ((32, 32, 32), (0, 0, 0), (32, 32, 32)),
    ((96, 8, 8), (0, 0, 0), (96, 6, 5)),
    ((96, 8, 8), (3, 1, 0), (80, 5, 4)),
]


@pytest.mark.parametrize("ng,e0,ne", HEX)
def test_hex_runs(cuda, monkeypatch, ng, e0, ne):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    Ad = generate_matrix(HexBlock(ng, e0, ne, h=1.0 / ng[0]), device=cuda)
    A = Ad.to_scipy()
    del Ad
    want, _ = _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2"), expect_runs=True)
    # every run lies inside one x-row, between its two end nodes
    nxf = ne[0] + 1 - (1 if e0[0] == 0 else 0)
    rows = A.shape[0] // 3 // nxf
    assert want <= rows * (nxf - 2)
    if ne[0] >= 64:
        assert want >= 0.8 * rows * (nxf - 2)


def test_hex_default_plan_reports_runs(cuda, monkeypatch):
    """Without any switch a 48^3 box takes the dictionary with runs, and the stream shrinks accordingly."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    _env(monkeypatch, {})
    A = generate_matrix(HexBlock((48,) * 3, (0, 0, 0), (48,) * 3, h=1.0 / 48), device=cuda)
    share = A.value_dict_run_share()
    assert 0.8 < share <= 46 / 48 + 1e-12, share
    nblk = A.nnz // 9
    assert A.stream_bytes() < A.spmv_bytes() * 0.05, (A.stream_bytes(), nblk)
    _env(monkeypatch, {"PCGB_SPMV_VDICT": "0"})
    from pcg_mpi_solver_b200.csr import CsrMatrix
    M = CsrMatrix(A.rowptr, A.col, A.val, A.shape)
    assert M.value_dict_run_share() == 0.0


# ------------------------------------------------------------------------------------------------ synthetic chains
def _chain(nn, reach=(-1, 0, 1), ids=None, one=None, shift=None, drop=None, seed=0):
    """A node chain: node i couples to i + r for r in reach (inside [0, nn)); block t takes the value of its offset's
    index t, so every interior node repeats its predecessor.  ids[i] = k adds k to every value index of node i; one = set
    of nodes whose middle block alone takes another value; shift[i] = s moves every column of node i by s nodes (breaks
    the +3 positions only); drop = set of nodes that lose their last block (breaks the block count only)."""
    rng = np.random.default_rng(seed)
    nbrs, vid = [], []
    for i in range(nn):
        off = np.array(reach) + (shift.get(i, 0) if shift else 0)
        cols = i + off
        keep = (cols >= 0) & (cols < nn)
        if drop and i in drop:
            keep[np.nonzero(keep)[0][-1]] = False
        nbrs.append(cols[keep])
        v = np.nonzero(keep)[0] + (0 if ids is None else ids.get(i, 0))
        if one and i in one:
            v[v.size // 2] = len(reach) + 4
        vid.append(v)
    A = C.node_block(nbrs, nn, rng)
    dic = rng.standard_normal((len(reach) + 5, 9))
    pos = _block_positions(A)
    A.data[pos] = dic[np.concatenate(vid)]
    return A


def _tile_nodes(A, tile):
    return C.tile_row_starts(A.indptr, tile, unit=3) // 3


@pytest.mark.parametrize("tile", ["300", "600", "1200", "3000"])
def test_chain_runs_across_tiles(cuda, monkeypatch, tile):
    """One long run cut by every tile boundary: runs that start and end exactly at a tile start / end; with 3000-item
    tiles a run is longer than 32 nodes, so more than one lane pass covers it."""
    A = _chain(700)
    want, _ = _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE=tile), expect_runs=True)
    starts = _tile_nodes(A, int(tile))
    if tile == "3000":
        assert np.diff(starts).max() > 64
    assert want >= 700 - 2 - 2 * (starts.size - 1)


@pytest.mark.parametrize("kind", ["id", "position", "count", "pairs"])
def test_run_breaks(cuda, monkeypatch, kind):
    """Runs broken only by one block id, only by a position one triple off, only by a block count; and runs of two."""
    nn = 400
    if kind == "id":
        A = _chain(nn, one=set(range(5, nn - 2, 9)))
    elif kind == "position":
        A = _chain(nn, reach=(-2, 0, 2), shift={i: 1 for i in range(6, nn - 3, 11)})
    elif kind == "count":
        A = _chain(nn, reach=(-2, -1, 0, 1, 2), drop=set(range(10, nn - 3, 7)))
    else:
        A = _chain(nn, ids={i: (i // 2) % 2 for i in range(nn)})   # node pairs (2k, 2k+1) share ids, the next pair differs
    tile = "300" if kind == "pairs" else "600"   # runs of two: 10-node tiles stay within the segment cap
    want, _ = _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE=tile), expect_runs=True)
    assert want < nn - 2


def test_segment_cap_falls_back(cuda, monkeypatch):
    """Runs of two separated by id changes: a tile of more than 8 segments is stored explicitly (no runs counted)."""
    nn = 600
    A = _chain(nn, ids={i: (i // 2) % 2 for i in range(nn)})
    want, _ = _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="2400"))
    uncapped = expected_run_nodes(A, 2400, cap=10**9)
    assert uncapped > 0 and want < uncapped


def test_no_runs(cuda, monkeypatch):
    """Every node differs from its predecessor in a block id: no runs, share 0, products unchanged."""
    nn = 500
    A = _chain(nn, ids={i: 2 * (i % 2) for i in range(nn)})
    want, _ = _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="600"), expect_runs=False)
    assert want == 0


def test_random_repeats(cuda, monkeypatch):
    """Random patterns and a small dictionary (tests/spmv_cases): few or no runs, exact either way."""
    A = _with_dictionary(C.nb_mixed().tocsr(), 3, seed=11)
    _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="600"))


# ------------------------------------------------------------------------------------------------ plan variants
# PCGB_SPMV_STAGES sets the ring of the value-streaming plan too, so the tiles are kept small enough for 8 of its stages
VARIANTS = [{"PCGB_BSR_CW": cw, "PCGB_SPMV_CTAS": c} for cw in (6, 8, 12) for c in (1, 2)] + [
    {"PCGB_SPMV_STAGES": s} for s in (2, 4, 8, 12)]


@pytest.mark.parametrize("index64", [False, True])
@pytest.mark.parametrize("var", VARIANTS, ids=lambda v: "-".join(f"{k[5:]}{x}" for k, x in v.items()))
def test_plan_variants(cuda, monkeypatch, var, index64):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    Ad = generate_matrix(HexBlock((40, 40, 40), (0, 3, 2), (30, 9, 8), h=1.0 / 40), device=cuda)
    A = Ad.to_scipy()
    del Ad
    _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="1500", **{k: str(v) for k, v in var.items()}),
           expect_runs=True, index64=index64)
    B = _chain(900, reach=(-3, -1, 0, 1, 3), one=set(range(11, 900, 17)))
    _check(monkeypatch, B, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="900", **{k: str(v) for k, v in var.items()}),
           expect_runs=True, index64=index64)


# ------------------------------------------------------------------------------------------------ full size
def test_256_box_run_share(cuda, monkeypatch):
    """256^3 (64-bit offsets): the run share is the x-rows' interior nodes less at most two per tile boundary.  The
    products of this box are compared bit for bit with PCGB_SPMV_VDICT=0 in test_gpu_spmv_vdict.py."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 70e9:
        pytest.skip("needs ~70 GB of free device memory")
    _env(monkeypatch, {})
    B = 256
    A = generate_matrix(HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B), device=cuda)
    assert A.rowptr.dtype == torch.int64 and A.value_dict_blocks() >= 1
    nn = A.shape[0] // 3
    rows = nn // B
    upper = rows * (B - 2)
    covered = A.value_dict_run_share() * nn
    assert upper - 2 * A.plan_info()["ntiles"] - 1 <= covered <= upper + 1e-6 * nn, (covered, upper)


# ------------------------------------------------------------------------------------------------ solves
@pytest.fixture(scope="module")
def box64(cuda):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, load_vector
    blk = HexBlock((64,) * 3, (0, 0, 0), (64,) * 3, h=1.0 / 64)
    return blk, generate_matrix(blk, device=cuda), load_vector(blk, device=cuda)


def _solve(monkeypatch, box, env, mg):
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk, A, b = box
    _env(monkeypatch, env)
    M = CsrMatrix(A.rowptr, A.col, A.val, A.shape)
    op = SubdomainOperator(M)
    pre = HexMultigrid(op, blk) if mg else op.jacobi()
    x, info = op.solve(b, pre, 0.0, 40, fixed_iters=True, record_resvec=True, trace=True, check_every=5)
    return M.value_dict_blocks(), M.value_dict_run_share(), x, info


@pytest.mark.parametrize("mg", [False, True])
def test_pcg_64_bit_identical(box64, monkeypatch, mg):
    import torch
    vd, share, x, info = _solve(monkeypatch, box64, {}, mg)
    vd0, share0, x0, info0 = _solve(monkeypatch, box64, {"PCGB_SPMV_VDICT": "0"}, mg)
    assert vd >= 1 and share > 0.8 and vd0 == 0 and share0 == 0.0
    assert torch.equal(_bits(x), _bits(x0))
    assert np.array_equal(info.resvec.view(np.int64), info0.resvec.view(np.int64))
    assert info.trace.tobytes() == info0.trace.tobytes() and info.iters == info0.iters == 40
