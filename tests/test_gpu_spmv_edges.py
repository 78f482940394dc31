"""Every SpMV kernel entrywise at its tile, node and 64-bit-offset edges, and its fused p.q epilogue inside PCG.

KERNELS is the kernel-forcing table: each entry is a set of PCGB_SPMV_* / PCGB_BSR_* variables and the plan_info() fields
it must produce.  Every test asserts the plan before it checks values, so a silent fall-back to another kernel fails.
Products go into a NaN-filled output (a row the kernel does not write shows) and are compared entrywise with a long-double
reference: |y - y_ref| <= 1e-13 (|A| |x|)_i, and x.y within 1e-12 sum_i |x_i| (|A| |x|)_i.  The matrices come from
tests/spmv_cases.py.  The fused dot of the persistent kernels is checked through spmv_split(with_dot=True); that of the
other kernels, and the split-row carries, only act inside the solver, so those entries solve against ref_pcg."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import spmv_cases as C

pytestmark = pytest.mark.gpu

RTOL = 1e-13        # as test_gpu_spmv.RTOL: fp64 summation-order noise only
DOT_RTOL = 1e-12
X_RTOL = 1e-10      # as test_gpu_pcg: solution parity with ref_pcg at tol 1e-13
ITER_SLACK = 2
TOL, MAXITER = 1e-13, 3000

_ROW = dict(index_mode=0, snap=1, split=False, tma=1)
_SPLIT = dict(index_mode=0, snap=0, split=True, tma=1)
_BSR = dict(index_mode=2, snap=1, split=False, tma=1, staged=2)
_GATE = {"PCGB_BSR_MIN_UNIFORM_PCT": "0"}   # small matrices are mostly boundary: keep the regularity gate out of it

KERNELS = {
    "ldg": ({"PCGB_SPMV_TMA": "0"}, dict(_ROW, staged=0, tma=0)),
    "tma": ({"PCGB_SPMV_STAGE": "0"}, dict(_ROW, staged=0)),
    "staged": ({"PCGB_SPMV_PERSIST": "0"}, dict(_ROW, staged=1)),
    "persist": ({"PCGB_SPMV_BSR": "0", "PCGB_SPMV_T3": "0"}, dict(_ROW, staged=2)),
    "t3": ({"PCGB_SPMV_BSR": "0", "PCGB_SPMV_T3": "1"}, dict(_ROW, staged=2, index_mode=1)),
    "split-persist": ({"PCGB_SPMV_SNAP": "0"}, dict(_SPLIT, staged=2)),
    "split-staged": ({"PCGB_SPMV_SNAP": "0", "PCGB_SPMV_PERSIST": "0"}, dict(_SPLIT, staged=1)),
    "split-merge": ({"PCGB_SPMV_SNAP": "0", "PCGB_SPMV_STAGE": "0"}, dict(_SPLIT, staged=0)),
    "long-rows": ({"PCGB_SPMV_BSR": "0"}, dict(_SPLIT, staged=2)),   # no SNAP variable: rows longer than a quarter tile split
}
for _u in (1, 0):
    for _i in (1, 0):
        for _cw in (6, 8, 12):
            KERNELS[f"bsr-uni{_u}-inplace{_i}-cw{_cw}"] = (
                dict(_GATE, PCGB_BSR_UNI=str(_u), PCGB_BSR_INPLACE=str(_i), PCGB_BSR_CW=str(_cw)), _BSR)
KERNELS["bsr-stages2-ctas2"] = (dict(_GATE, PCGB_SPMV_STAGES="2", PCGB_SPMV_CTAS="2"), _BSR)
KERNELS["bsr-stages4-ctas1"] = (dict(_GATE, PCGB_SPMV_STAGES="4", PCGB_SPMV_CTAS="1"), _BSR)
BSR_ENTRIES = [k for k in KERNELS if k.startswith("bsr-")]

# case name -> (builder, PCGB_SPMV_TILE or None); built once per session (seeded)
CASES = {
    "nb-empty": (lambda: C.nb_empty()[0], 1200),
    "nb-singleton": (C.nb_singleton, None),
    "nb-mixed": (C.nb_mixed, 900),
    "nb-1-node": (lambda: C.nb_small(1), None),
    "nb-2-nodes": (lambda: C.nb_small(2), None),
    "nb-1-tile": (lambda: C.nb_small(40), None),
    "nb-many": (C.nb_many, 600),
    "nb-rect": (C.nb_rect, None),
    "rg-empty-rows": (C.rg_empty_rows, None),
    "rg-windows": (C.rg_windows, 1024),
    "rg-long-1024": (lambda: C.rg_long_rows(1024), 1024),
    "rg-long-256": (lambda: C.rg_long_rows(256), 256),
    "hex": (lambda: R.hex_box_csr((9, 7, 5), (0, 0, 0), (9, 7, 5)), None),
}
for _L in (4, 8, 16, 32):
    CASES[f"rg-lengths-{_L}"] = (functools.partial(C.rg_lengths, _L), None)
    CASES[f"rg-triples-{_L}"] = (functools.partial(C.rg_triples, _L), None)
for _m in C.BSR_MAX_ROW.values():      # longest node at the node-block limit and one block above it (default tile)
    for _b in (_m // 3, _m // 3 + 1):
        CASES[f"nb-banded-{_b}"] = (functools.partial(C.nb_banded, _b), None)

NODE_CASES = ["nb-empty", "nb-singleton", "nb-mixed", "nb-1-node", "nb-2-nodes", "nb-1-tile", "nb-many", "nb-rect"]


@functools.lru_cache(maxsize=None)
def _case(name):
    """(A, x, y_ref, scale) of a case; x is seeded by the name."""
    A = CASES[name][0]().tocsr()
    x = np.random.default_rng(sum(map(ord, name))).standard_normal(A.shape[1])
    y_ref, scale = C.ref_spmv(A, x)
    return A, x, y_ref, scale


def _force(monkeypatch, env, tile=None):
    """Exactly `env` (plus the tile) among the SpMV plan variables."""
    for k in list(os.environ):
        if k.startswith("PCGB_SPMV_") or k.startswith("PCGB_BSR_"):
            monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    if tile:
        monkeypatch.setenv("PCGB_SPMV_TILE", str(tile))


def _assert_plan(info, want):
    for k, v in want.items():
        got = info["split_rows"] > 0 if k == "split" else info[k]
        assert got == v, (k, v, info)


def _nan(n, dev):
    import torch
    return torch.full((n,), float("nan"), dtype=torch.float64, device=dev)


def _assert_entrywise(y, y_ref, scale, what):
    y = np.asarray(y)
    assert not np.isnan(y).any(), (what, "rows not written", np.nonzero(np.isnan(y))[0][:10])
    err = np.abs(y.astype(np.longdouble) - y_ref) / (scale + 1e-300)
    assert float(err.max(initial=0.0)) <= RTOL, (what, float(err.max()), int(err.argmax()))


def _dot_bound(x, y_ref, scale):
    return float(np.sum(x.astype(np.longdouble) * y_ref)), DOT_RTOL * float(np.abs(x) @ scale) + 1e-300


def _run(cuda, entry, name, lanes_key=None, lanes=None):
    """Both row-offset widths of one table entry on one case: plan, NaN-filled y against the reference, int32 == int64 bit
    for bit, and for persistent plans without split rows the fused dot through spmv_split.  Returns the int32 plan."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    A, x, y_ref, scale = _case(name)
    want = dict(KERNELS[entry][1])
    if lanes_key:
        want["lanes"] = lanes
    xd = torch.from_numpy(x).to(cuda)
    ys, infos = [], []
    for idx64 in (False, True):
        M = CsrMatrix.from_scipy(A, device=cuda, index64=idx64)
        assert M.rowptr.dtype == (torch.int64 if idx64 else torch.int32)
        info = M.plan_info()
        _assert_plan(info, want)
        y = M.spmv(xd, out=_nan(A.shape[0], cuda))
        _assert_entrywise(y.cpu().numpy(), y_ref, scale, (entry, name, idx64))
        if info["staged"] == 2 and info["split_rows"] == 0 and A.shape[0] == A.shape[1]:
            M.set_boundary_rows(torch.arange(0, A.shape[0], 7, dtype=torch.int32, device=cuda))
            y2, d = M.spmv_split(xd, with_dot=True, out=_nan(A.shape[0], cuda))
            assert torch.equal(y2, y), (entry, name, idx64)
            d_ref, bound = _dot_bound(x, y_ref, scale)
            assert abs(float(d) - d_ref) <= bound, (entry, name, idx64, float(d), d_ref)
        ys.append(y)
        infos.append(info)
    assert torch.equal(ys[0], ys[1]), (entry, name, "int32 and int64 row offsets differ")
    return infos[0]


def _tile_starts(name, info, unit):
    A = _case(name)[0]
    return A, C.tile_row_starts(A.indptr, info["tile_items"], unit)


# ------------------------------------------------------------------------------------------------ row-group kernels
@pytest.mark.parametrize("lanes", [4, 8, 16, 32])
@pytest.mark.parametrize("entry", ["ldg", "tma", "staged", "persist"])
def test_row_group_kernels(cuda, monkeypatch, entry, lanes):
    for name in (f"rg-lengths-{lanes}", "rg-empty-rows", "rg-windows", "nb-mixed"):
        _force(monkeypatch, dict(KERNELS[entry][0], PCGB_SPMV_LANES=str(lanes)), CASES[name][1])
        info = _run(cuda, entry, name, "lanes", lanes)
        if name == "rg-windows" and info["staged"]:
            assert info["max_windows_per_tile"] > 32, info
        if name == "rg-empty-rows":
            A, s = _tile_starts(name, info, 1)
            empty = np.diff(A.indptr) == 0
            assert empty[s[1:-1]].any(), "no tile starts at an empty row"
            assert any(s[b + 1] > s[b] and A.indptr[s[b + 1]] == A.indptr[s[b]] for b in range(len(s) - 1)), "no all-empty tile"


@pytest.mark.parametrize("lanes3", [4, 8, 16, 32])
def test_triple_index_kernel(cuda, monkeypatch, lanes3):
    for name in (f"rg-triples-{lanes3}", "hex"):
        _force(monkeypatch, dict(KERNELS["t3"][0], PCGB_SPMV_LANES3=str(lanes3)))
        _run(cuda, "t3", name, "lanes", lanes3)


@pytest.mark.parametrize("entry", ["split-persist", "split-staged", "split-merge", "long-rows"])
def test_split_row_kernels(cuda, monkeypatch, entry):
    names = ["rg-long-1024", "rg-long-256"] + (["rg-empty-rows", "nb-mixed"] if entry != "long-rows" else [])
    for name in names:
        _force(monkeypatch, KERNELS[entry][0], CASES[name][1])
        info = _run(cuda, entry, name)
        if name.startswith("rg-long"):
            assert info["max_row"] > 3 * info["tile_items"], info        # one row spans more than 3 tiles


# ------------------------------------------------------------------------------------------------ node-block kernel
@pytest.mark.parametrize("entry", BSR_ENTRIES)
def test_node_block_kernel(cuda, monkeypatch, entry):
    import torch
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    for name in NODE_CASES:
        _force(monkeypatch, KERNELS[entry][0], CASES[name][1])
        info = _run(cuda, entry, name)
        if name == "nb-empty":
            A, s = _tile_starts(name, info, 3)
            empty_node = C.blocks_per_node(A) == 0
            assert empty_node[s[1:-1] // 3].any(), "no tile starts at an empty node"
            assert any(s[b + 1] > s[b] and A.indptr[s[b + 1]] == A.indptr[s[b]] for b in range(len(s) - 1)), "no tile without blocks"
        if name in ("nb-1-node", "nb-2-nodes", "nb-1-tile"):
            assert info["ntiles"] == 1, info
        if name == "nb-singleton":
            assert 1 < info["ntiles"] < sms, info                           # fewer tiles than resident CTAs
        if name == "nb-many":
            assert info["ntiles"] >= 6 * info["resident_ctas"], info      # every stage of every CTA's ring wraps


@pytest.mark.parametrize("inplace", [1, 0])
def test_node_block_max_row_limit(cuda, monkeypatch, inplace):
    """The longest node just inside the node-block limit keeps the kernel; one block more drops it (row-group kernel)."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    below = C.BSR_MAX_ROW[inplace] // 3                     # blocks of the long node: 3 * blocks non-zeros per row
    _force(monkeypatch, dict(_GATE, PCGB_BSR_INPLACE=str(inplace)))
    for blocks, want in ((below, 2), (below + 1, 0)):
        name = f"nb-banded-{blocks}"
        A, x, y_ref, scale = _case(name)
        for idx64 in (False, True):
            M = CsrMatrix.from_scipy(A, device=cuda, index64=idx64)
            info = M.plan_info()
            assert info["index_mode"] == want and info["max_row"] == 3 * blocks, info
            y = M.spmv(torch.from_numpy(x).to(cuda), out=_nan(A.shape[0], cuda))
            _assert_entrywise(y.cpu().numpy(), y_ref, scale, (name, inplace, idx64))


# ------------------------------------------------------------------------------------------------ inside the solver
SOLVE_ENTRIES = ["ldg", "tma", "staged", "persist", "t3", "split-persist", "split-staged", "split-merge"] + BSR_ENTRIES


@functools.lru_cache(maxsize=None)
def _spd(kind):
    A = {"poisson": lambda: R.poisson27(12), "hex": lambda: R.hex_box_csr((9, 7, 5), (0, 0, 0), (9, 7, 5)),
         "node": C.nb_spd, "poisson48": lambda: R.poisson27(48)}[kind]().tocsr()
    b = A @ np.random.default_rng(21).standard_normal(A.shape[0])
    minv = 1.0 / A.diagonal()
    hist = []
    ref = R.ref_pcg([R.CsrPart(A, b)], [minv], TOL, MAXITER, resvec=hist)
    assert ref["Flag"] == 0 and ref["Iter"] > 12
    return A, b, minv, ref, np.array(hist)


def _solve_matches_oracle(M, kind, batching=True):
    from pcg_mpi_solver_b200 import solve
    A, b, minv, ref, hist = _spd(kind)
    x, flag, relres, iters, info = solve(M, b, minv, TOL, MAXITER, check_every=1, use_graph=False, record_resvec=True,
                                         return_info=True)
    assert flag == ref["Flag"] == 0 and abs(iters - ref["Iter"]) <= ITER_SLACK, (flag, iters, ref["Iter"])
    np.testing.assert_allclose(info.resvec[:12], hist[:12], rtol=1e-9)      # a wrong p.q changes alpha in iteration 1
    assert np.linalg.norm(x - ref["X"][0]) <= X_RTOL * np.linalg.norm(ref["X"][0])
    if batching:
        for check_every, graph in ((1, True), (7, False), (7, True)):
            got = solve(M, b, minv, TOL, MAXITER, check_every=check_every, use_graph=graph)
            assert got[1:] == (flag, relres, iters), (check_every, graph)
            assert np.array_equal(got[0], x), (check_every, graph)


@pytest.mark.parametrize("entry", SOLVE_ENTRIES)
def test_fused_dot_in_solver(cuda, monkeypatch, entry):
    """Every kernel's p.q epilogue (and the split-row carries) inside PCG against ref_pcg, int32 and int64 row offsets,
    with check_every 1 / 7 and graph on / off bit-identical."""
    from pcg_mpi_solver_b200.csr import CsrMatrix
    kind = "node" if entry.startswith("bsr-") else "hex" if entry == "t3" else "poisson"
    _force(monkeypatch, KERNELS[entry][0])
    for idx64 in (False, True):
        M = CsrMatrix.from_scipy(_spd(kind)[0], device=cuda, index64=idx64)
        _assert_plan(M.plan_info(), KERNELS[entry][1])
        _solve_matches_oracle(M, kind)


def test_stage_reduce_of_many_dot_partials(cuda, monkeypatch):
    """More than 8192 per-tile p.q partials (one CTA per tile, 256-item tiles) go through the solver's staged reduction."""
    from pcg_mpi_solver_b200.csr import CsrMatrix
    _force(monkeypatch, {"PCGB_SPMV_PERSIST": "0"}, 256)
    M = CsrMatrix.from_scipy(_spd("poisson48")[0], device=cuda)
    info = M.plan_info()
    assert info["staged"] == 1 and info["ntiles"] > 8192, info
    _solve_matches_oracle(M, "poisson48", batching=False)


# ------------------------------------------------------------------------------------------------ TMA alignment fall-back
@pytest.mark.parametrize("which", ["val", "col"])
def test_unaligned_arrays_fall_back(cuda, monkeypatch, which):
    """TMA bulk copies need 16-byte aligned sources: a CsrMatrix over views one element into their storage runs the plain
    load kernel (no staged or node-block kernel), computes the same, and solves."""
    import torch
    from pcg_mpi_solver_b200.csr import CsrMatrix
    _force(monkeypatch, _GATE)
    A, b, minv, ref, hist = _spd("hex")
    rp = torch.from_numpy(A.indptr.astype(np.int32)).to(cuda)
    arrays = {"col": torch.from_numpy(A.indices.astype(np.int32)).to(cuda), "val": torch.from_numpy(A.data.copy()).to(cuda)}
    assert CsrMatrix(rp, arrays["col"], arrays["val"], A.shape).plan_info()["index_mode"] == 2   # aligned: node-block kernel
    t = arrays[which]
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=cuda)
    buf[1:] = t
    arrays[which] = buf[1:]
    assert arrays[which].data_ptr() % 16 != 0
    M = CsrMatrix(rp, arrays["col"], arrays["val"], A.shape)
    assert M.val.data_ptr() == arrays["val"].data_ptr() and M.col.data_ptr() == arrays["col"].data_ptr()
    info = M.plan_info()
    assert info["tma"] == 0 and info["index_mode"] == 0 and info["staged"] == 0, info
    x = np.random.default_rng(5).standard_normal(A.shape[0])
    y_ref, scale = C.ref_spmv(A, x)
    y = M.spmv(torch.from_numpy(x).to(cuda), out=_nan(A.shape[0], cuda))
    _assert_entrywise(y.cpu().numpy(), y_ref, scale, which)
    _solve_matches_oracle(M, "hex", batching=False)


# ------------------------------------------------------------------------------------------------ offsets above 2^31
def test_block256_int64_offsets(cuda):
    """The 256^3 box of `bench.py --block 256` (4.08e9 non-zeros, int64 row offsets) on the node-block kernel: sampled rows
    against a long-double recomputation from the device CSR arrays (a few thousand consecutive rows on each side of the rows
    whose offsets cross 2^31 and 3 * 2^30, the first and the last rows; tile boundaries are not exposed, so the windows are
    wide), and the symmetry w.(A x) = x.(A w).  nnz < 2^32, so no offset crosses 2^32; the last rows carry the largest."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 60e9:
        pytest.skip("needs ~60 GB of free device memory")
    blk = HexBlock((256, 256, 256), (0, 0, 0), (256, 256, 256), h=1.0 / 256)
    A = generate_matrix(blk, device=cuda)
    n, nnz = A.shape[0], A.nnz
    assert A.rowptr.dtype == torch.int64 and 2**31 < nnz < 2**32
    info = A.plan_info()
    assert info["index_mode"] == 2 and info["staged"] == 2 and info["split_rows"] == 0, info
    g = torch.Generator(device=cuda).manual_seed(3)
    x = torch.randn(n, dtype=torch.float64, device=cuda, generator=g)
    w = torch.randn(n, dtype=torch.float64, device=cuda, generator=g)
    y = A.spmv(x, out=_nan(n, cuda))
    cross = torch.searchsorted(A.rowptr, torch.tensor([2**31, 3 * 2**30], dtype=torch.int64, device=cuda), right=True) - 1
    half = 3000
    wins = [(0, half), (n - half, n)] + [(max(0, r - half), min(n, r + half)) for r in cross.tolist()]
    xh = x.cpu().numpy()
    for a, e in wins:
        rp = A.rowptr[a:e + 1].cpu().numpy()
        k0, k1 = int(rp[0]), int(rp[-1])
        cols = A.col[k0:k1].cpu().numpy()
        vals = A.val[k0:k1].cpu().numpy()
        S = sp.csr_matrix((vals, cols, rp - k0), shape=(e - a, n))
        prod = np.append(S.data.astype(np.longdouble) * xh[S.indices].astype(np.longdouble), np.longdouble(0))
        y_ref = np.add.reduceat(prod, np.minimum(S.indptr[:-1], S.nnz))
        scale = abs(S) @ np.abs(xh)
        _assert_entrywise(y[a:e].cpu().numpy(), y_ref, scale, (a, e, k0, k1))
    assert any(int(A.rowptr[r]) <= 2**31 < int(A.rowptr[r + 1]) for r in cross.tolist()[:1])
    Ax = y.clone()
    Aw = A.spmv(w)
    s1, s2 = float(torch.dot(w, Ax)), float(torch.dot(x, Aw))
    assert abs(s1 - s2) <= 1e-11 * float(w.norm() * Ax.norm()), (s1, s2)
    del A, x, w, y, Ax, Aw
    torch.cuda.empty_cache()
