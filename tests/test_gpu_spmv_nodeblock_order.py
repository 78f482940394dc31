"""The node-block SpMV against an exact restatement of its row order (tests/nodeblock_cases.py), at every ring, group and
run-segment edge its plan can choose.

A node-block tile is a whole number of nodes, so y does not depend on the plan: every case compares y of `spmv` and of the
split launch (interface tiles first), each written into a NaN-filled output, bit for bit with `rows_f64`, and the fused
x.y with the exact dot within (n + 2) 2^-53 sum |x_r y_r|, on the dictionary kernel and with PCGB_SPMV_VDICT=0.  The ring
the plan reports (CsrMatrix.value_dict_plan) must be the host restatement's, the stream size the host count of words."""
import functools
import time

import numpy as np
import pytest

from tests import nodeblock_cases as N
from tests import spmv_cases as C
from tests.test_gpu_spmv_vdict import _GATE, _env, _tensors, _with_dictionary

pytestmark = pytest.mark.gpu
RINGS = set()   # (stages, group, producers, consumers) of every dictionary plan this file checked
DOT_ERR = [0.0]  # largest |x.y - exact| / sum |x_r y_r| of the fused dot


@pytest.fixture(scope="module", autouse=True)
def _runtime(request):
    t0 = time.time()
    yield
    rep = request.config.pluginmanager.get_plugin("terminalreporter")
    msg = (f"test_gpu_spmv_nodeblock_order.py: {time.time() - t0:.1f} s, largest dot error {DOT_ERR[0]:.3e} of sum |x_r y_r|, "
           f"rings reached {sorted(RINGS)}")
    if rep is not None:
        rep.write_line(msg)
    else:
        print(msg)


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Hand the test's device memory back to the driver: the 128^3 and 256^3 boxes leave tens of GB in torch's cache,
    which later tests that check free memory (cudaMemGetInfo) would otherwise not see."""
    yield
    import gc

    import torch
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


def _assert_rows(got, want, what):
    bad = np.nonzero(_bits(got) != _bits(want))[0]
    assert bad.size == 0, f"{what}: {bad.size} rows differ, first {bad[:5]}: {got[bad[:5]]} against {want[bad[:5]]}"


def _run(M, x_dev, boundary):
    """(y, y of the split launch, fused x.y) on NaN-filled outputs."""
    import torch
    n = M.shape[0]
    y = torch.full((n,), float("nan"), dtype=torch.float64, device=x_dev.device)
    M.spmv(x_dev, out=y)
    M.set_boundary_rows(boundary)
    ys = torch.full_like(y, float("nan"))
    _, d = M.spmv_split(x_dev, with_dot=True, out=ys)
    torch.cuda.synchronize()
    return y.cpu().numpy(), ys.cpu().numpy(), float(d.item())


def _boundary(n, seed):
    import torch
    rng = np.random.default_rng(seed)
    return torch.from_numpy(np.unique(rng.integers(0, max(n, 1), max(n // 50, 1))).astype(np.int32)).cuda()


def _check_dot(d, x, y):
    exact, s = N.exact_dot(x, y)
    assert abs(d - exact) <= (y.size + 2) * N.EPS * s, (d, exact, s)
    if s > 0:
        DOT_ERR[0] = max(DOT_ERR[0], abs(d - exact) / s)


def _plan(M):
    info, vp = M.plan_info(), M.value_dict_plan()
    return info, vp, M.value_dict_blocks()


def _check_ring(M, env_stages=0):
    """The plan's ring equals vd_ring of the plan's own caps; returns (info, vd plan, D)."""
    info, vp, vd = _plan(M)
    assert vd >= 1 and all(vp[k] > 0 for k in ("stages", "group", "producers", "consumers", "cap_words", "cap_nodes", "ctas_per_sm")), vp
    r = N.vd_ring(info["x_cap"], vp["cap_nodes"], vp["cap_words"], vd, vp["consumers"], vp["ctas_per_sm"], env_stages)
    assert r is not None and (vp["stages"], vp["group"], vp["producers"]) == (r["stages"], r["group"], r["producers"]), (vp, r)
    assert info["smem_bytes"] == r["smem"], (info["smem_bytes"], r)
    assert vp["stages"] % vp["producers"] == 0 and vp["group"] <= vp["stages"] <= N.MAX_STAGES
    RINGS.add((vp["stages"], vp["group"], vp["producers"], vp["consumers"]))
    return info, vp, vd


def _check_stream(M, A, info, vp, vd):
    """nvwords and cap_words against k_vd_runs restated on the plan's tiles; stream_bytes against the host count."""
    starts = C.tile_row_starts(A.indptr, info["tile_items"], unit=3) // 3
    assert starts.size - 1 == info["ntiles"]
    _, words, covered = N.vd_runs(A, starts)
    nvw, cap = N.stream_words(words)
    assert (vp["nvwords"], vp["cap_words"]) == (nvw, cap), (vp, nvw, cap)
    assert M.value_dict_run_share() == covered.sum() / (A.shape[0] // 3)
    rp64 = M.rowptr.dtype.itemsize == 8
    assert M.stream_bytes() == N.stream_bytes(info, vd, nvw, A.shape[0], A.shape[1], rp64)


def _check(monkeypatch, A, env, x=None, seed=0, index64=False, ring=True, stream=False, want_vd=True):
    """Products of the plan under env and under env + PCGB_SPMV_VDICT=0 against rows_f64; the ring and optionally the
    stream size of the dictionary plan.  Returns (info, vd plan, D) of the plan under env."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    A = A.tocsr()
    x = N.signed_x(A.shape[1], seed) if x is None else x
    want = N.rows_f64(A, x)
    rp, col, val = _tensors(A, "cuda", index64=index64)
    xd = torch.from_numpy(x).cuda()
    boundary = _boundary(A.shape[0], seed)
    out = None
    for e in (env, dict(env, PCGB_SPMV_VDICT="0")):
        _env(monkeypatch, e)
        M = CsrMatrix(rp, col, val, A.shape)
        if e is env:
            if want_vd:
                out = _check_ring(M, int(e.get("PCGB_SPMV_STAGES", 0))) if ring else _plan(M)
                if stream:
                    _check_stream(M, A, *out)
            else:
                out = _plan(M)
        else:
            assert M.value_dict_blocks() == 0
        y, ys, d = _run(M, xd, boundary)
        _assert_rows(y, want, f"spmv {e}")
        _assert_rows(ys, want, f"spmv_split {e}")
        _check_dot(d, x, want)
        del M
    return out


# ------------------------------------------------------------------------------------------------ order pin
@pytest.mark.parametrize("index64", [False, True])
@pytest.mark.parametrize("tile", [None, "300"])
def test_order_pin(cuda, monkeypatch, index64, tile):
    """Rows whose bits hold only in the documented order (block order, fma nesting, +0.0 start), on both consumers."""
    A, x, kinds = N.order_pin()
    env = dict(_GATE, PCGB_SPMV_VDICT="2")
    if tile:
        env["PCGB_SPMV_TILE"] = tile
    _, _, vd = _check(monkeypatch, A, env, x=x, index64=index64)
    assert vd >= 5


# ------------------------------------------------------------------------------------------------ rings
@functools.lru_cache(maxsize=1)
def _nb_many():
    return C.nb_many().tocsr()


def _many(nd):
    return _with_dictionary(_nb_many(), nd, seed=nd)


FORCED = [1, 3, 5, 6, 7, 10, 14, 16, 17]


@pytest.mark.parametrize("stages", FORCED)
def test_forced_rings(cuda, monkeypatch, stages):
    """PCGB_SPMV_STAGES: 1 and 3 stages (as many producers), odd rings (1 producer), 6 / 10 / 14 (2), 16 (4), 17 -> 16."""
    env = dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="600")
    _, vp, _ = _check(monkeypatch, _many(37), dict(env, PCGB_SPMV_STAGES=str(stages)), stream=stages in (1, 17))
    assert vp["stages"] == min(stages, 16) and vp["group"] == min(6, stages) and vp["producers"] == N.producers(min(stages, 16))


def _classes_by_nd(caps, cw, ctas):
    """Dictionary sizes 1..1024 grouped by the default ring they give with the probe plan's caps."""
    cls = {}
    for nd in range(1, 1025):
        r = N.vd_ring(caps[0], caps[1], caps[2], nd, cw, ctas)
        if r is None:
            continue
        k = "deepest" if r["group"] == cw and r["stages"] == min(2 * cw + 2, 16) else \
            "g+2" if r["group"] == cw and r["stages"] == cw + 2 else "g<cw" if r["group"] < cw else "between"
        cls.setdefault(k, []).append(nd)
    return cls


DEFAULT_CLASSES = {}   # class -> (cw, ctas, nd) reached


@pytest.mark.parametrize("cw", [6, 8, 12])
@pytest.mark.parametrize("ctas", [1, 2])
def test_default_rings(cuda, monkeypatch, cw, ctas):
    """The default search, CW x CTAs per SM, at dictionary sizes that land on G = CW with the deepest ring, on G = CW with
    G + 2 stages and on G < CW (chosen from the caps of a probe plan; the getter must equal the restatement)."""
    from pcg_mpi_solver_b200.csr import CsrMatrix
    env = dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="1500", PCGB_BSR_CW=str(cw), PCGB_SPMV_CTAS=str(ctas))
    A = _many(1)
    rp, col, val = _tensors(A, "cuda")
    _env(monkeypatch, env)
    M = CsrMatrix(rp, col, val, A.shape)
    info, vp, _ = _check_ring(M)
    del M
    caps = (info["x_cap"], vp["cap_nodes"], vp["cap_words"])
    cls = _classes_by_nd(caps, cw, vp["ctas_per_sm"])
    for k in ("deepest", "g+2", "g<cw"):
        if k not in cls:
            continue
        nd = cls[k][len(cls[k]) // 2]
        _, vp, vd = _check(monkeypatch, _many(nd), env, seed=nd, stream=k == "g<cw")
        assert vd == nd and vp["consumers"] == cw
        got = "deepest" if vp["group"] == cw and vp["stages"] == min(2 * cw + 2, 16) else \
            "g+2" if vp["group"] == cw and vp["stages"] == cw + 2 else "g<cw" if vp["group"] < cw else "between"
        DEFAULT_CLASSES.setdefault(got, []).append((cw, ctas, nd))


def test_every_ring_class_was_reached(cuda, monkeypatch):
    """Together the forced and default cases reach every (producers, stages) class of the dictionary ring."""
    for s in FORCED:
        if not any(r[0] == min(s, 16) for r in RINGS):
            test_forced_rings(cuda, monkeypatch, s)
    for cw in (6, 8, 12):
        for ctas in (1, 2):
            if not any(c[:2] == (cw, ctas) for v in DEFAULT_CLASSES.values() for c in v):
                test_default_rings(cuda, monkeypatch, cw, ctas)
    have = {(s, p) for s, _, p, _ in RINGS}
    for need in [(1, 1), (3, 3), (6, 2), (10, 2), (14, 2), (16, 4)]:
        assert need in have, (need, sorted(RINGS))
    assert any(s >= 5 and s % 2 == 1 and p == 1 for s, p in have), sorted(RINGS)
    assert any(g < s and s % g != 0 for s, g, _, _ in RINGS), sorted(RINGS)   # a ring that is not a whole number of groups
    for k in ("deepest", "g+2", "g<cw"):
        assert k in DEFAULT_CLASSES, DEFAULT_CLASSES


# ------------------------------------------------------------------------------------------------ fallbacks
def test_forced_ring_that_does_not_fit(cuda, monkeypatch):
    """A forced ring too large for the plan's CTAs per SM: no dictionary, run share 0, and exactly the plan (and stream
    bytes) of PCGB_SPMV_VDICT=0 under the same switches."""
    from pcg_mpi_solver_b200.csr import CsrMatrix
    env = dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE="1200", PCGB_BSR_CW="12", PCGB_SPMV_CTAS="2", PCGB_SPMV_STAGES="16")
    probe = dict(env, PCGB_SPMV_STAGES="2")
    A = _many(1)
    rp, col, val = _tensors(A, "cuda")
    _env(monkeypatch, probe)
    M = CsrMatrix(rp, col, val, A.shape)
    info, vp, _ = _plan(M)
    del M
    _env(monkeypatch, dict(env, PCGB_SPMV_VDICT="0"))
    M0 = CsrMatrix(rp, col, val, A.shape)
    ctas16 = M0.plan_info()["resident_ctas"]
    del M0
    nds = [nd for nd in range(1, 1025) if N.vd_ring(info["x_cap"], vp["cap_nodes"], vp["cap_words"], nd, 12, 2, 16) is None]
    assert nds, "no dictionary size makes a 16-stage ring overflow two CTAs"
    nd = nds[len(nds) // 2]
    B = _many(nd)
    info, _, vd = _check(monkeypatch, B, env, seed=nd, want_vd=False)
    assert vd == 0 and ctas16 > 0
    rp, col, val = _tensors(B, "cuda")
    _env(monkeypatch, env)
    M = CsrMatrix(rp, col, val, B.shape)
    _env(monkeypatch, dict(env, PCGB_SPMV_VDICT="0"))
    M0 = CsrMatrix(rp, col, val, B.shape)
    assert M.value_dict_blocks() == 0 and M.value_dict_run_share() == 0.0
    assert M.value_dict_plan() == dict.fromkeys(M.value_dict_plan(), 0)
    assert M.plan_info() == M0.plan_info() and M.stream_bytes() == M0.stream_bytes()
    assert M.plan_info()["index_mode"] == 2


@pytest.mark.parametrize("delta", [-1, 0])
def test_mode1_refusal_boundary(cuda, monkeypatch, delta):
    """PCGB_SPMV_VDICT=1 refuses a dictionary of D blocks when the matrix has fewer than 2 D x grid blocks: block-diagonal
    matrices of exactly 2 D grid - 1 (refused) and 2 D grid (taken) blocks."""
    from pcg_mpi_solver_b200.csr import CsrMatrix
    env = dict(_GATE, PCGB_SPMV_TILE="300")
    nd = 24
    A = C.nb_singleton(nn=30000).tocsr()
    rp, col, val = _tensors(A, "cuda")
    _env(monkeypatch, dict(env, PCGB_SPMV_VDICT="0"))
    grid = CsrMatrix(rp, col, val, A.shape).plan_info()["resident_ctas"]
    nn = 2 * nd * grid + delta
    B = _with_dictionary(C.nb_singleton(nn=nn).tocsr(), nd, seed=nn)
    info, _, vd = _check(monkeypatch, B, dict(env, PCGB_SPMV_VDICT="1"), seed=nn, want_vd=delta == 0, ring=True)
    assert info["resident_ctas"] == grid and info["ntiles"] > grid, (info, grid)
    assert vd == (nd if delta == 0 else 0)


# ------------------------------------------------------------------------------------------------ stream size
def _chain(**kw):
    from tests.test_gpu_spmv_vdict_runs import _chain as chain
    return chain(**kw)


@pytest.mark.parametrize("case,tile", [("run", "300"), ("run", "3000"), ("id", "600"), ("position", "600"), ("count", "600"),
                                       ("pairs", "300"), ("cap", "2400"), ("none", "600")])
def test_stream_size_chains(cuda, monkeypatch, case, tile):
    nn = 400
    A = {"run": lambda: _chain(nn=700), "id": lambda: _chain(nn=nn, one=set(range(5, nn - 2, 9))),
         "position": lambda: _chain(nn=nn, reach=(-2, 0, 2), shift={i: 1 for i in range(6, nn - 3, 11)}),
         "count": lambda: _chain(nn=nn, reach=(-2, -1, 0, 1, 2), drop=set(range(10, nn - 3, 7))),
         "pairs": lambda: _chain(nn=nn, ids={i: (i // 2) % 2 for i in range(nn)}),
         "cap": lambda: _chain(nn=600, ids={i: (i // 2) % 2 for i in range(600)}),
         "none": lambda: _chain(nn=500, ids={i: 2 * (i % 2) for i in range(500)})}[case]()
    _check(monkeypatch, A, dict(_GATE, PCGB_SPMV_VDICT="2", PCGB_SPMV_TILE=tile), seed=len(case), stream=True)


# ------------------------------------------------------------------------------------------------ hex boxes
BOXES = [  # (ng, e0, ne): e0 == 0 has the clamped face; cubes and slabs, x-rows shorter and longer than a tile
    ((20, 20, 20), (0, 0, 0), (20, 20, 20)),
    ((33, 33, 33), (3, 2, 1), (27, 25, 23)),
    ((48, 48, 48), (0, 0, 0), (48, 48, 48)),
    ((160, 24, 8), (0, 0, 0), (160, 20, 6)),
    ((160, 160, 8), (5, 0, 0), (150, 140, 4)),
    ((16, 160, 40), (0, 0, 0), (14, 150, 36)),
    ((11, 160, 160), (0, 0, 0), (9, 150, 150)),
    ((64, 64, 64), (0, 0, 0), (64, 64, 64)),
]
FULL = 48 ** 3 * 1.1


def _sampled_rows(Md, starts_nodes, nrows, extra, rng):
    """Rows around tile starts, the first and last rows, `extra` and random ones."""
    t = starts_nodes[rng.choice(starts_nodes.size, min(starts_nodes.size, 1500), replace=False)] * 3
    rows = np.concatenate([t - 3, t - 1, t, t + 2, t + 3, [0, 1, 2, nrows - 3, nrows - 1], extra, rng.integers(0, nrows, 3000)])
    return np.unique(rows[(rows >= 0) & (rows < nrows)])


def _device_rows(M, rows):
    """(indptr, indices, data) of the sampled rows, read from the device arrays."""
    import torch
    r = torch.from_numpy(rows).cuda()
    a, e = M.rowptr[r].long(), M.rowptr[r + 1].long()
    cnt = e - a
    take = torch.repeat_interleave(a - torch.cumsum(cnt, 0) + cnt, cnt) + torch.arange(int(cnt.sum()), device=r.device)
    ip = np.concatenate([[0], np.cumsum(cnt.cpu().numpy())])
    return ip, M.col[take].cpu().numpy(), M.val[take].cpu().numpy()


def _check_box(monkeypatch, Md, blk, seed, full):
    """Default plan of a generated box: ring, stream (full boxes), y and the split launch against rows_f64 (all rows or
    sampled ones), x.y against the exact dot of the device y."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    n = Md.shape[0]
    x = N.signed_x(Md.shape[1], seed)
    xd = torch.from_numpy(x).cuda()
    boundary = _boundary(n, seed)
    indptr = Md.rowptr.cpu().numpy()
    out = None
    for e in ({}, {"PCGB_SPMV_VDICT": "0"}):
        _env(monkeypatch, e)
        M = CsrMatrix(Md.rowptr, Md.col, Md.val, Md.shape)
        if not e:
            out = _check_ring(M)
            info = out[0]
            starts = C.tile_row_starts(indptr, info["tile_items"], unit=3) // 3
            nxf = blk.ne[0] + 1 - (1 if blk.e0[0] == 0 else 0)
            face = np.arange(0, n // 3, nxf) * 3 if blk.e0[0] == 0 else np.zeros(0, np.int64)   # next to the clamped face
            if full:
                A = M.to_scipy()
                _check_stream(M, A, *out)
                want = N.rows_f64(A, x)
                rows = None
            else:
                rows = _sampled_rows(M, starts, n, np.concatenate([face[:2000], face[:2000] + 1]), np.random.default_rng(seed))
                want = N.rows_f64_csr(*_device_rows(M, rows), x)
        else:
            assert M.value_dict_blocks() == 0
        y, ys, d = _run(M, xd, boundary)
        _assert_rows(y if rows is None else y[rows], want, f"spmv {e}")
        _assert_rows(ys if rows is None else ys[rows], want, f"spmv_split {e}")
        assert not np.isnan(y).any() and np.array_equal(_bits(y), _bits(ys))
        _check_dot(d, x, y)
        del M
    return out


@pytest.mark.parametrize("ng,e0,ne", BOXES, ids=lambda v: "x".join(map(str, v)))
def test_default_plans_over_boxes(cuda, monkeypatch, ng, e0, ne):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    blk = HexBlock(ng, e0, ne, h=1.0 / max(ng))
    _env(monkeypatch, {})
    Md = generate_matrix(blk, device=cuda)
    assert Md.plan_info()["index_mode"] == 2 and Md.value_dict_blocks() >= 1, Md.plan_info()
    info, vp, vd = _check_box(monkeypatch, Md, blk, seed=sum(ne), full=Md.shape[0] / 3 <= FULL)
    print(f"box {ng} {e0} {ne}: tile {info['tile_items']}, {Md.shape[0] / 3 / info['ntiles']:.1f} nodes per tile, ring {vp}")


def test_box_plans_cover_tile_shapes(cuda, monkeypatch):
    """The boxes keep the default tile and have x-rows shorter and longer than a tile.  Where the planner shrinks the tile
    (6-node x-rows: two CTAs of two value-streaming stages do not fit), it ends on the row-group plan, not on this kernel."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    row_short = row_long = False
    for ng, e0, ne in BOXES + [((8, 160, 160), (0, 0, 0), (6, 150, 150))]:
        _env(monkeypatch, {})
        Md = generate_matrix(HexBlock(ng, e0, ne, h=1.0 / max(ng)), device=cuda)
        info = Md.plan_info()
        shrunk = info["tile_items"] < 6100 - 3 * (info["max_row"] + 1)
        if ne[0] == 6:
            assert shrunk and info["index_mode"] != 2 and Md.value_dict_blocks() == 0, info
            continue
        assert not shrunk and info["index_mode"] == 2, info
        per_tile = Md.shape[0] / 3 / info["ntiles"]
        nxf = ne[0] + 1 - (1 if e0[0] == 0 else 0)
        row_short |= nxf < per_tile
        row_long |= nxf > per_tile
        del Md
    assert row_short and row_long


def test_box_128(cuda, monkeypatch):
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 24e9:
        pytest.skip("needs ~20 GB of free device memory")
    blk = HexBlock((128,) * 3, (0, 0, 0), (128,) * 3, h=1.0 / 128)
    _env(monkeypatch, {})
    Md = generate_matrix(blk, device=cuda)
    info, vp, vd = _check_box(monkeypatch, Md, blk, seed=128, full=False)
    print(f"128^3: info {info} ring {vp} D {vd}")
    # DESIGN: G = 6 and 12 stages (4 producer warps), 105 216 B per CTA, two CTAs per SM
    assert (vp["stages"], vp["group"], vp["producers"], vp["consumers"], vp["ctas_per_sm"]) == (12, 6, 4, 6, 2), vp
    assert info["smem_bytes"] == 105216


def test_box_256_past_2_31(cuda, monkeypatch):
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 70e9:
        pytest.skip("needs ~70 GB of free device memory")
    B = 256
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    _env(monkeypatch, {})
    Md = generate_matrix(blk, device=cuda)
    assert Md.rowptr.dtype == torch.int64
    r31 = int(torch.searchsorted(Md.rowptr, torch.tensor([2 ** 31], dtype=torch.int64, device=cuda)).item())
    x = N.signed_x(Md.shape[1], 256)
    xd = torch.from_numpy(x).cuda()
    _check_ring(Md)
    y = torch.full((Md.shape[0],), float("nan"), dtype=torch.float64, device=cuda)
    Md.spmv(xd, out=y)
    rows = np.arange(max(r31 - 900, 0), min(r31 + 900, Md.shape[0]))
    indptr = Md.rowptr.cpu().numpy()
    starts = C.tile_row_starts(indptr, Md.plan_info()["tile_items"], unit=3) // 3
    rows = np.unique(np.concatenate([rows, _sampled_rows(Md, starts, Md.shape[0], np.zeros(0, np.int64), np.random.default_rng(2))]))
    want = N.rows_f64_csr(*_device_rows(Md, rows), x)
    _assert_rows(y.cpu().numpy()[rows], want, "256^3")
