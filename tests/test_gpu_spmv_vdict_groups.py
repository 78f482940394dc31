"""The dictionary consumer of the node-block SpMV (spmv.cuh k_spmv_bsr3_vd) takes a CTA's tiles in groups of G, one warp
per tile, and stores the group's rows after one barrier.  y, the split launch and its fused x.y must be the same bits as
the kernel that streams the values (PCGB_SPMV_VDICT=0) whatever the consumer warps, the CTAs per SM, the tiles left over
after the last whole group, and the nodes and rows of a tile past one warp and past all consumer threads."""
import numpy as np
import pytest

from tests import spmv_cases as C
from tests.test_gpu_spmv_vdict import _GATE, _assert_same_bits, _env, _bits, _tensors, _with_dictionary

pytestmark = pytest.mark.gpu


def _check(dev, monkeypatch, A, env, seed=0):
    """Bit-identical to VDICT=0 (y, split y, split x.y) and entrywise against the long-double product."""
    rp, col, val = _tensors(A, dev)
    vd, info, info0, (x, y) = _assert_same_bits(monkeypatch, rp, col, val, A.shape, dict(_GATE, PCGB_SPMV_VDICT="2", **env), seed)
    assert vd > 0 and info["index_mode"] == 2 and info["staged"] == 2
    assert info["ntiles"] == info0["ntiles"] and info["resident_ctas"] == info0["resident_ctas"]
    y_ref, scale = C.ref_spmv(A, x.cpu().numpy())
    err = np.abs(y.cpu().numpy().astype(np.longdouble) - y_ref) / (scale + 1e-300)
    assert float(err.max(initial=0.0)) <= 1e-13
    return info


@pytest.mark.parametrize("ctas", [1, 2])
@pytest.mark.parametrize("cw", [6, 8, 12])
def test_consumer_warps_and_ctas(cuda, monkeypatch, cw, ctas):
    A = _with_dictionary(C.nb_many().tocsr(), 61, seed=cw + ctas)
    for tile in (None, "600"):
        env = {"PCGB_BSR_CW": str(cw), "PCGB_SPMV_CTAS": str(ctas)}
        if tile:
            env["PCGB_SPMV_TILE"] = tile
        _check(cuda, monkeypatch, A, env, seed=cw)


@pytest.mark.parametrize("cw", [6, 12])
def test_tiles_left_after_the_last_group(cuda, monkeypatch, cw):
    """PCGB_SPMV_STAGES=4 gives groups of G = min(CW, 4) = 4 tiles.  Tile sizes are chosen until some CTA ends with a
    whole number of groups, some with one tile past the last group and some with G - 1."""
    G = 4
    A = _with_dictionary(C.nb_many().tocsr(), 37, seed=11)
    want, seen = {0, 1, G - 1}, set()
    from pcg_mpi_solver_b200.csr import CsrMatrix
    rp, col, val = _tensors(A, cuda)
    for tile in range(300, 1200, 18):
        env = {"PCGB_BSR_CW": str(cw), "PCGB_SPMV_CTAS": "1", "PCGB_SPMV_STAGES": "4", "PCGB_SPMV_TILE": str(tile)}
        _env(monkeypatch, dict(_GATE, PCGB_SPMV_VDICT="2", **env))
        info = CsrMatrix(rp, col, val, A.shape).plan_info()
        nt, grid = info["ntiles"], info["resident_ctas"]
        res = {(nt // grid) % G} | ({(nt // grid + 1) % G} if nt % grid else set())
        if res - seen:
            _check(cuda, monkeypatch, A, env, seed=tile)
            seen |= res
        if want <= seen:
            break
    assert want <= seen, seen


def test_fewer_tiles_than_ctas(cuda, monkeypatch):
    A = _with_dictionary(C.nb_small(40).tocsr(), 9, seed=2)
    info = _check(cuda, monkeypatch, A, {"PCGB_SPMV_TILE": "300"})
    assert 1 < info["ntiles"] == info["resident_ctas"], info   # the grid is cut to the tiles


@pytest.mark.parametrize("cw", [6, 12])
def test_tile_past_one_warp_and_all_consumer_threads(cuda, monkeypatch, cw):
    """Single-block nodes (12 merge items each) in tiles of 4000 items: over 300 nodes and 900 rows per tile, more
    than the 32 lanes of the owning warp walk and more than the CW * 32 consumer threads store."""
    A = _with_dictionary(C.nb_singleton(nn=6001).tocsr(), 23, seed=cw)
    info = _check(cuda, monkeypatch, A, {"PCGB_BSR_CW": str(cw), "PCGB_SPMV_TILE": "4000"})
    assert info["tile_items"] == 4000 and 3 * (info["tile_items"] // 12) > cw * 32 + 32, info


@pytest.mark.parametrize("cw", [8, 12])
def test_pcg_64_bit_identical(cuda, monkeypatch, cw):
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock((64,) * 3, (0, 0, 0), (64,) * 3, h=1.0 / 64)
    A = generate_matrix(blk, device=cuda)
    b = load_vector(blk, device=cuda)
    out = []
    for vdict in ("1", "0"):
        _env(monkeypatch, {"PCGB_BSR_CW": str(cw), "PCGB_SPMV_VDICT": vdict})
        M = CsrMatrix(A.rowptr, A.col, A.val, A.shape)
        op = SubdomainOperator(M)
        x, info = op.solve(b, op.jacobi(), 0.0, 40, fixed_iters=True, record_resvec=True)
        out.append((M.value_dict_blocks(), x.clone(), info))
        del op, M
    (vd, x, info), (vd0, x0, info0) = out
    assert vd > 0 and vd0 == 0
    assert torch.equal(_bits(x), _bits(x0))
    assert np.array_equal(info.resvec.view(np.int64), info0.resvec.view(np.int64)) and info.iters == info0.iters == 40
