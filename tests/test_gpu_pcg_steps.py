"""The PCG iteration step by step against its own reductions, and every exit path of the control logic.

Each solve records the loop trace (`SubdomainOperator.solve(trace=..., snapshot=...)`): one record per control step with
the reduced values it consumed and the control block after it.  tests/pcg_shadow.py replays the records and must
reproduce every field bit for bit.  Solves with fixed_iters and maxiter = k, k = 1..K, then give the vectors after every
iteration, and each step is checked entrywise against a long-double restatement:
    p = Minv r (iteration 0, exact) or fma(beta, p, Minv r)         within 1 ulp
    r = r - alpha q,  x = x + alpha p (into the buffer the shadow predicts; a frozen XMin stays untouched)   1 ulp
    q = A p                                                        within 1e-13 (|A||p|)_i
    pp, xx (x before the update), rr, rz, p.q                      within (count+2) 2^-53 sum|terms|;  #inf(z) exact
With x0 given, r0 = b - A x0 is in no snapshot, so p of iteration 0 is then checked through q, p.q and the sums only.
The recorded residual history must equal the norms the shadow computes from the same records, entry by entry.
"""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import pcg_cases as C
from tests import pcg_shadow as S

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
LD = np.longdouble


def _op(A, cuda, n_global=None):
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    return SubdomainOperator(CsrMatrix.from_scipy(sp.csr_matrix(A), device=cuda), n_global=n_global)


def _t(v, cuda):
    import torch
    return None if v is None else torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _solve(op, c, cuda, **kw):
    args = dict(x0=_t(c.get("x0"), cuda), w=_t(c.get("w"), cuda), max_stag=c.get("max_stag", 3))
    args.update(kw)
    args.setdefault("record_resvec", True)
    x, info = op.solve(_t(c["b"], cuda), _t(c.get("minv"), cuda), c["tol"], c["maxiter"], trace=True, snapshot=True, **args)
    return x.cpu().numpy(), info


def _replay(info, c, fixed=False):
    sh = S.replay(info.trace, c["tol"], c["maxiter"], c["n_global"], c.get("max_stag", 3), fixed_iters=fixed)
    res = sh.result
    assert res is not None and info.trace_total == len(info.trace)
    assert (res["flag"], res["iters"], res["imin"], res["stag"], res["moresteps"], res["too_small_tol"]) == \
        (info.flag, info.iters, info.imin, info.stag, info.moresteps, info.too_small_tol)
    assert S.same_bits(res["relres"], info.relres)
    if info.resvec is not None:       # ||r_0||, then the recurrence's ||r|| of every iteration at index iter + 1
        assert S.same_bits(info.resvec[0], np.sqrt(float(info.trace[0]["inp"][S.R0R0])))
        for i, v in sh.resvec.items():
            assert S.same_bits(info.resvec[i], v), (i, info.resvec[i], v)
    return sh


def _fma_close(got, a, b, c):
    """got is a*b + c rounded once (fma), within 1 ulp of the result plus the long-double reference's own rounding of the
    product and the sum (which dominates where a*b and c cancel)."""
    ab = LD(a) * b.astype(LD) if np.isscalar(a) else a.astype(LD) * b.astype(LD)
    ref = ab + c.astype(LD)
    bound = np.spacing(np.abs(ref.astype(np.float64))) + LD(2.0 ** -62) * (np.abs(ab) + np.abs(c.astype(LD)))
    return np.all(np.abs(got.astype(LD) - ref) <= bound)


def _within(got, ref_ld, terms_abs_sum, count):
    bound = (count + 2) * U * terms_abs_sum
    return abs(LD(got) - ref_ld) <= bound


# ------------------------------------------------------------------------------------------- every exit path
EXIT = C.exit_cases()


@pytest.mark.parametrize("name", sorted(EXIT))
def test_exit_path_reached_and_replayed(cuda, name):
    c = EXIT[name]
    op = _op(c["A"], cuda, c["n_global"])
    x, info = _solve(op, c, cuda)
    assert c["path"](info.trace), (name, [int(k) for k in info.trace["kind"]])
    ref = C.ref_solve(c)
    assert info.flag == ref["Flag"], (name, info.flag, ref["Flag"])
    if c["margin"]:
        assert info.iters == ref["Iter"], (name, info.iters, ref["Iter"])
    if c["too_small"] is not None:
        assert info.too_small_tol == c["too_small"] == bool(ref["too_small_tol"]), name
    if len(info.trace) == 0:     # early exit: the initial guess comes back unchanged
        x0 = c["x0"] if c["x0"] is not None else np.zeros_like(c["b"])
        assert np.array_equal(x, x0)
        return
    sh = _replay(info, c)
    snap = info.snapshot
    assert int(snap["xcur"]) == int(info.trace[-1]["ctrl"]["xcur"]) and int(snap["alias"]) == int(info.trace[-1]["ctrl"]["alias"])
    xo = snap["x"][sh.result["xout"]]
    assert np.array_equal(x, xo, equal_nan=True)          # the buffer the finalisation picks
    if name == "converge_first_verify":                     # after the verification: r = b - q exactly, q = A x_cur
        xc = snap["x"][int(snap["xcur"])]
        assert np.array_equal(snap["r"], c["b"] - snap["q"])
        Aq = c["A"].astype(np.longdouble) @ xc.astype(np.longdouble)
        assert np.all(np.abs(snap["q"] - Aq) <= 1e-13 * (abs(c["A"]) @ np.abs(xc)) + 1e-300)


def test_flag1_finalisation_branches_and_alias(cuda):
    """Flag 1 with XMin still aliased to X and after it was frozen, and both finalisation branches, over a scan of maxiter."""
    H = R.hex_box_csr((5, 4, 4), (0, 0, 0), (5, 4, 4))
    b = np.random.default_rng(8).standard_normal(H.shape[0])
    D = sp.diags(np.tile([1.0, 100.0], 25)).tocsr()      # the first step multiplies ||r|| by ~5: XMin stays bound to X
    scans = [(D, np.tile([10.0, 1.0], 25), None, mi) for mi in (1, 2)] + [(H, b, 1.0 / H.diagonal(), mi) for mi in range(1, 41)]
    seen = set()
    for A_, b_, m_, mi in scans:
        op = _op(A_, cuda)
        c = C.case(A_, b_, minv=m_, tol=1e-30, maxiter=mi)
        x, info = _solve(op, c, cuda)
        assert info.flag == C.ref_solve(c)["Flag"] == 1
        _replay(info, c)
        fin = info.trace[-1]
        normr_min = np.sqrt(fin["inp"][S.RR])
        seen.add((int(fin["ctrl"]["alias"]), bool(normr_min < fin["ctrl"]["normr_act"])))
        assert np.array_equal(x, info.snapshot["x"][int(fin["ctrl"]["xmin"])])
    assert {a for a, _ in seen} == {0, 1}, seen
    assert {br for _, br in seen} == {False, True}, seen


def test_failed_verification_then_moresteps_then_convergence(cuda):
    """A failed verification, MoreSteps > 0 iterations verified one by one, then convergence (found by a scan of tol on the
    device; the reference is solved with the same tol and must give the same flag)."""
    A = R.poisson27(10)
    b = A @ np.random.default_rng(5).standard_normal(A.shape[0])
    op = _op(A, cuda, n_global=C.BIG)
    found = None
    for tol in np.geomspace(1e-13, 1e-17, 60):
        c = C.case(A, b, minv=1.0 / A.diagonal(), tol=float(tol), maxiter=2000, n_global=C.BIG)
        x, info = _solve(op, c, cuda)
        kinds = [int(k) for k in info.trace["kind"]]
        ver = [r for r in info.trace if int(r["kind"]) == S.VERIFY]
        if info.flag == 0 and len(ver) >= 2 and int(ver[-1]["ctrl"]["moresteps"]) >= 1:
            found = (c, info, kinds)
            break
    assert found is not None, "no tol in the scan fails a verification and then converges"
    c, info, kinds = found
    _replay(info, c)
    # after the first failed verification every iteration is verified: ITER, VERIFY, RESUME, ITER, VERIFY, ...
    first = kinds.index(S.VERIFY)
    tail = kinds[first:-1]
    assert tail[0::3] == [S.VERIFY] * len(tail[0::3]) and all(k == S.RESUME for k in tail[1::3])
    assert C.ref_solve(c)["Flag"] == 0


def test_last_iteration_ends_in_failed_verification(cuda):
    """maxiter reached right after a failed verification: the head that follows finds the loop exhausted (flag 1)."""
    A = R.poisson27(6)
    b = A @ np.random.default_rng(6).standard_normal(A.shape[0])
    op = _op(A, cuda, n_global=C.BIG)
    c = C.case(A, b, minv=1.0 / A.diagonal(), tol=1e-19, maxiter=2000, n_global=C.BIG)
    _, info = _solve(op, c, cuda)
    first_verify_iter = int(next(r for r in info.trace if int(r["kind"]) == S.VERIFY)["ctrl"]["iter"])
    c = C.case(A, b, minv=1.0 / A.diagonal(), tol=1e-19, maxiter=first_verify_iter + 1, n_global=C.BIG)
    _, info = _solve(op, c, cuda)
    kinds = [int(k) for k in info.trace["kind"]]
    assert kinds[-3:] == [S.VERIFY, S.RESUME, S.FINAL] and int(info.trace[-2]["ctrl"]["state"]) == S.ST_EXHAUSTED
    assert info.flag == C.ref_solve(c)["Flag"] == 1
    _replay(info, c)


# ------------------------------------------------------------------------------------------- step identities
def _band(n):
    """Cheap SPD band matrix (diagonally dominant, 5 diagonals)."""
    if n == 1:
        return sp.csr_matrix(np.array([[3.0]]))
    diags = [np.full(n, 4.0), np.full(n - 1, -1.0), np.full(n - 1, -1.0)]
    offs = [0, -1, 1]
    if n > 2:
        diags += [np.full(n - 2, -0.5), np.full(n - 2, -0.5)]
        offs += [-2, 2]
    return sp.diags(diags, offs).tocsr()


def _cap():
    import torch
    return min(8 * torch.cuda.get_device_properties(0).multi_processor_count, 2048) * 1024


def _inputs(n, kind_minv, kind_x0, kind_w, seed):
    rng = np.random.default_rng(seed)
    A = _band(n)
    b = rng.standard_normal(n)
    minv = 1.0 / A.diagonal() * rng.uniform(0.5, 1.5, n) if kind_minv else None
    x0 = rng.standard_normal(n) if kind_x0 else None
    w = {"none": None, "random": rng.uniform(0.1, 1.0, n), "partition": 1.0 / rng.choice([1.0, 2.0, 4.0, 8.0], n)}[kind_w]
    return A, b, minv, x0, w


def _check_steps(cuda, A, b, minv, x0, w, K, use_graph=True, check_every=16):
    n = A.shape[0]
    op = _op(A, cuda)
    c = C.case(A, b, minv=minv, x0=x0, w=w, tol=1e-30, maxiter=1)
    Aabs = abs(A)
    wv = np.ones(n) if w is None else w
    prev = None
    for k in range(1, K + 1):
        c["maxiter"] = k
        _, info = _solve(op, c, cuda, fixed_iters=True, use_graph=use_graph, check_every=check_every)
        _replay(info, c, fixed=True)
        tr, snap = info.trace, info.snapshot
        nit = [int(t) for t in tr["kind"]].count(S.ITER)
        if nit < k:      # a tiny system solved exactly: rho = 0 at the head of iteration k-1, nothing new ran
            assert nit == k - 1 and int(tr[nit]["ctrl"]["state"]) == S.ST_BREAK and int(tr[nit]["ctrl"]["flag"]) == 4
            return
        assert [int(t) for t in tr["kind"]] == [S.HEAD] + [S.ITER] * k + [S.FINAL]
        if int(tr[k - 1]["ctrl"]["state"]) == S.ST_BREAK:      # an exactly solved tiny system broke down at a head
            return
        rec = tr[k]                       # iteration k-1
        it = k - 1
        broke = int(rec["ctrl"]["state"]) == S.ST_BREAK
        if broke and int(rec["ctrl"]["iter"]) == it:     # stopped at alpha: the update did not run
            return
        alpha = float(rec["ctrl"]["alpha"])
        p, q, r = snap["p"], snap["q"], snap["r"]
        if prev is None:
            # p = Minv r0 (r0 = b bit for bit when no x0 is given)
            if x0 is None:
                assert np.array_equal(p, minv * b if minv is not None else b)
            rprev = None
        else:
            ptr, psnap = prev
            # the shorter run's trace is a prefix of this one: every record before its last iteration bit for bit but for the
            # maxiter field, and the inputs of that iteration (its control block ends in EXHAUSTED there, not in the next head)
            a, b_ = tr[:k - 1].copy(), ptr[:k - 1].copy()
            assert np.all(a["ctrl"]["maxiter"] == k) and np.all(b_["ctrl"]["maxiter"] == k - 1)
            a["ctrl"]["maxiter"] = b_["ctrl"]["maxiter"] = 0
            assert a.tobytes() == b_.tobytes()
            assert tr[k - 1]["inp"].tobytes() == ptr[k - 1]["inp"].tobytes()
            beta = float(tr[k - 1]["ctrl"]["beta"])               # set by the head of iteration `it`
            rprev = psnap["r"]
            z = minv * rprev if minv is not None else rprev
            assert _fma_close(p, beta, psnap["p"], z)
            assert _fma_close(r, -alpha, q, rprev)
            # x into the buffer predicted from the control block before the iteration; a frozen XMin stays untouched
            cb = tr[k - 1]["ctrl"]
            cur = int(cb["xcur"])
            dst = cur ^ 1 if (not int(cb["alias"]) and cur == int(cb["xmin"])) else cur
            xs = psnap["x"][cur]
            assert _fma_close(snap["x"][dst], alpha, p, xs)
            if dst != cur:
                assert np.array_equal(snap["x"][cur], xs)
            assert int(rec["ctrl"]["xcur"]) == dst
        # q = A p
        qref = A.astype(LD) @ p.astype(LD)
        assert np.all(np.abs(q - qref) <= 1e-13 * (Aabs @ np.abs(p)) + 1e-300)
        # the fused sums of this iteration against the snapshot vectors (x before its update)
        xs = (x0 if x0 is not None else np.zeros(n)) if prev is None else prev[1]["x"][int(tr[k - 1]["ctrl"]["xcur"])]
        z = minv * r if minv is not None else r
        for slot, t in ((S.PP, p * (p * wv)), (S.XX, xs * (xs * wv)), (S.RR, r * (r * wv)), (S.RZ, z * (r * wv)), (S.PQ, p * q)):
            tl = t.astype(LD)
            assert _within(rec["inp"][slot], tl.sum(), float(np.abs(tl).sum()), n), (k, slot)
        assert float(rec["inp"][S.NINF]) == float(np.isinf(z).sum())
        prev = (tr, snap)
        if broke:
            return


SMALL_N = [1, 2, 255, 256, 257, 1023, 1024, 1025]
COMBOS = [(m, x, w) for m in (True, False) for x in (False, True) for w in ("none", "random", "partition")]


@pytest.mark.parametrize("n", SMALL_N)
def test_steps_small_n(cuda, n):
    for j, (m, x, w) in enumerate(COMBOS):
        A, b, minv, x0, wv = _inputs(n, m, x, w, seed=100 * n + j)
        _check_steps(cuda, A, b, minv, x0, wv, K=25 if j < 4 else 8)


@pytest.mark.parametrize("edge", ["cap-1", "cap", "cap+1", "3cap+17"])
def test_steps_at_the_vector_grid_cap(cuda, edge):
    """n around 8 CTAs per SM x 1024: beyond it the grid-stride loops run more than once and k_reduce sums > 256 partials."""
    cap = _cap()
    n = {"cap-1": cap - 1, "cap": cap, "cap+1": cap + 1, "3cap+17": 3 * cap + 17}[edge]
    A, b, minv, x0, w = _inputs(n, True, edge != "cap", "random" if edge in ("cap", "3cap+17") else "partition", seed=7)
    _check_steps(cuda, A, b, minv, x0, w, K=3)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("check_every", [1, 7, 25])
def test_batching_gives_identical_traces(cuda, use_graph, check_every):
    A, b, minv, x0, w = _inputs(1025, True, True, "random", seed=11)
    c = C.case(A, b, minv=minv, x0=x0, w=w, tol=1e-30, maxiter=25)
    base_x, base = _solve(_op(A, cuda), c, cuda, fixed_iters=True, use_graph=False, check_every=1)
    x, info = _solve(_op(A, cuda), c, cuda, fixed_iters=True, use_graph=use_graph, check_every=check_every)
    assert info.trace.tobytes() == base.trace.tobytes() and np.array_equal(x, base_x)
    _check_steps(cuda, A, b, minv, x0, w, K=4, use_graph=use_graph, check_every=check_every)
    # a converging solve too: same trace whatever the batching
    c = C.case(A, b, minv=minv, x0=x0, w=w, tol=1e-10, maxiter=400)
    _, a = _solve(_op(A, cuda), c, cuda, use_graph=False, check_every=1)
    _, g = _solve(_op(A, cuda), c, cuda, use_graph=use_graph, check_every=check_every)
    assert a.trace.tobytes() == g.trace.tobytes()
    _replay(g, c)


def test_one_rank_weights_leave_pq_unweighted(cuda):
    """On one rank the device's p.q is the unweighted sum of p_i (A p)_i, while ref_pcg weights it (:487): documented in
    pcgb200.h.  Pinned here, with everything else of the iteration weighted."""
    A, b, minv, _, w = _inputs(2000, True, False, "random", seed=3)
    c = C.case(A, b, minv=minv, w=w, tol=1e-30, maxiter=1)
    _, info = _solve(_op(A, cuda), c, cuda, fixed_iters=True)
    p, q = info.snapshot["p"], info.snapshot["q"]
    pq = float(info.trace[1]["inp"][S.PQ])
    un, wd = (p * q).astype(LD), (p * q * w).astype(LD)
    assert _within(pq, un.sum(), float(np.abs(un).sum()), p.size)
    assert not _within(pq, wd.sum(), float(np.abs(wd).sum()), p.size)
    tr = []
    C.ref_solve(c, trace=tr)
    ref_pq = next(e["pq"] for e in tr if e["step"] == "pq")
    assert abs(ref_pq - float(wd.sum())) <= 1e-12 * abs(ref_pq)


# ------------------------------------------------------------------------------------------- capacity, handle reuse
def test_trace_capacity_drops_extra_records_and_writes_nothing_beyond(cuda):
    import ctypes

    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.solver import TRACE_DTYPE, TRACE_HEADER_BYTES
    A, b, minv, _, _ = _inputs(300, True, False, "none", seed=4)
    op = _op(A, cuda)
    c = C.case(A, b, minv=minv, tol=1e-30, maxiter=20)
    _, full = _solve(op, c, cuda, fixed_iters=True)
    assert full.trace_total == 22
    for cap in (0, 1, 5, 21):
        _, info = op.solve(_t(b, cuda), _t(minv, cuda), 1e-30, 20, trace=cap, fixed_iters=True)
        assert info.trace_total == 22 and len(info.trace) == cap
        assert info.trace.tobytes() == full.trace[:cap].tobytes()
        # a raw buffer with a guard region after the records: nothing is written past the capacity
        rb = TRACE_DTYPE.itemsize
        buf = torch.full((TRACE_HEADER_BYTES + (cap + 4) * rb,), 0xA5, dtype=torch.uint8, device=cuda)
        lib = _lib.load()
        _lib.check(lib.pcgb_solver_set_trace(op._solver, _lib.ptr(buf), cap, None))
        try:
            x = torch.zeros(A.shape[0], dtype=torch.float64, device=cuda)
            opt = _lib.Options(tol=1e-30, maxiter=20, n_global=A.shape[0], max_stag=3, check_every=16, use_graph=1, fixed_iters=1,
                               record_resvec=0, time_kernels=0, x0_zero=1)
            res = _lib.Result()
            _lib.check(lib.pcgb_solve(op._solver, _lib.ptr(_t(b, cuda)), _lib.ptr(_t(minv, cuda)), None, _lib.ptr(x), ctypes.byref(opt),
                                      None, ctypes.byref(res), _lib.stream_ptr()))
        finally:
            _lib.check(lib.pcgb_solver_set_trace(op._solver, None, 0, None))
        raw = buf.cpu().numpy()
        assert int(raw[:8].view(np.uint64)[0]) == 22
        assert np.all(raw[TRACE_HEADER_BYTES + cap * rb:] == 0xA5)


def test_handle_reuse_is_bit_identical_to_fresh_handles(cuda):
    """One operator solves a sequence that toggles M, w, resvec, trace, x0, check_every, tol, fixed_iters and max_stag;
    every result equals the same solve on a fresh operator bit for bit (graphs keyed on every captured argument)."""
    A, b, minv, x0, w = _inputs(3000, True, True, "random", seed=9)
    bt, mt, xt, wt = (_t(v, cuda) for v in (b, minv, x0, w))
    seq = [dict(M=mt, w=None, record_resvec=True, trace=True, x0=None, check_every=16, tol=1e-10, fixed_iters=False, max_stag=3),
           dict(M=None, w=wt, record_resvec=False, trace=False, x0=xt, check_every=7, tol=1e-12, fixed_iters=False, max_stag=2),
           dict(M=mt, w=wt, record_resvec=True, trace=False, x0=None, check_every=16, tol=1e-9, fixed_iters=True, max_stag=0),
           dict(M=mt, w=None, record_resvec=False, trace=True, x0=xt, check_every=1, tol=1e-11, fixed_iters=False, max_stag=1),
           dict(M=None, w=None, record_resvec=True, trace=True, x0=None, check_every=16, tol=1e-10, fixed_iters=True, max_stag=3),
           dict(M=mt, w=None, record_resvec=True, trace=True, x0=None, check_every=16, tol=1e-10, fixed_iters=False, max_stag=3)]
    shared = _op(A, cuda)
    for kw in seq:
        kw = dict(kw)
        M, tol = kw.pop("M"), kw.pop("tol")
        xa, ia = shared.solve(bt, M, tol, 60, **kw)
        xb, ib = _op(A, cuda).solve(bt, M, tol, 60, **kw)
        assert np.array_equal(xa.cpu().numpy(), xb.cpu().numpy())
        for f in ("flag", "iters", "relres", "imin", "stag", "moresteps", "too_small_tol", "matvecs"):
            assert getattr(ia, f) == getattr(ib, f), f
        if kw["record_resvec"]:
            assert np.array_equal(ia.resvec, ib.resvec)
        if kw["trace"]:
            assert ia.trace.tobytes() == ib.trace.tobytes() and len(ia.trace) > 0
        else:
            assert ia.trace is None


def test_reuse_with_only_the_weights_changed(cuda):
    """Two graph solves on one handle that differ in nothing but w: the second must not replay the first one's graph."""
    A, b, minv, _, w1 = _inputs(3000, True, False, "random", seed=12)
    w2 = 1.0 / np.random.default_rng(13).choice([1.0, 2.0, 4.0], A.shape[0])
    bt, mt = _t(b, cuda), _t(minv, cuda)
    wt = (_t(w1, cuda), _t(w2, cuda))          # both alive: distinct device addresses (a freed one could be handed out again)
    shared = _op(A, cuda)
    for w in (wt[0], wt[1], wt[0]):
        xa, ia = shared.solve(bt, mt, 1e-10, 200, w=w, check_every=16, use_graph=True, record_resvec=True)
        xb, ib = _op(A, cuda).solve(bt, mt, 1e-10, 200, w=w, check_every=16, use_graph=True, record_resvec=True)
        assert np.array_equal(xa.cpu().numpy(), xb.cpu().numpy()) and np.array_equal(ia.resvec, ib.resvec)
        assert (ia.flag, ia.iters, ia.relres) == (ib.flag, ib.iters, ib.relres)


def test_zz_report_stagnation_fma_disagreements():
    """How often the rounded and the exact evaluation of the stagnation test disagreed over every replay of this module
    (the device's record decides those; printed with -rP)."""
    print(f"stagnation tests replayed: {S.FMA_STATS['tests']}, rounded/exact disagreements: {S.FMA_STATS['disagreements']}")
