"""Seeded PCG problems that drive the control logic down each exit path (shared by the CPU shadow pin and the GPU tests).

Each case is a dict: A (scipy CSR), b, minv (None = no preconditioner), x0 (None = zero), tol, maxiter, n_global,
max_stag, and `path`, a predicate on the (device or reference-derived) record sequence that says the intended path was
taken.  `margin` is True where the problem is built so that no decision of the loop sits within rounding of its
threshold; there the iteration count must equal the reference's exactly.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests.pcg_shadow import FINAL, HEAD, ITER, PQ, RZ, ST_BREAK, ST_EXHAUSTED, VERIFY

BIG = 10 ** 7   # n_global large enough that MaxMSteps = 5


def _last(recs, kind):
    for r in reversed(recs):
        if int(r["kind"]) == kind:
            return r
    return None


def kinds(recs):
    return [int(r["kind"]) for r in recs]


def case(A, b, *, minv=None, x0=None, tol=1e-8, maxiter=100, n_global=None, max_stag=3, margin=False, path=None, w=None,
         too_small=None):
    """too_small: the expected TooSmallTolerance outcome (None = not asserted)."""
    A = sp.csr_matrix(A)
    return dict(A=A, b=np.asarray(b, float), minv=None if minv is None else np.asarray(minv, float),
                x0=None if x0 is None else np.asarray(x0, float), tol=tol, maxiter=maxiter,
                n_global=int(n_global if n_global is not None else A.shape[0]), max_stag=max_stag, margin=margin, path=path,
                w=None if w is None else np.asarray(w, float), too_small=too_small)


def _diag(d):
    return sp.diags(np.asarray(d, float)).tocsr()


def _stop_rec(recs):
    """The record of the step after which the loop stopped (a trigger hands over to the verification and is no stop)."""
    for r in recs:
        k, st = int(r["kind"]), int(r["ctrl"]["state"])
        if k == FINAL:
            break
        if st in (ST_BREAK, ST_EXHAUSTED) or (k == VERIFY and st != 0):
            return r
    return None


def _stop(recs):
    """(kind, flag, state) of the step after which the loop stopped."""
    r = _stop_rec(recs)
    return None if r is None else (int(r["kind"]), int(r["ctrl"]["flag"]), int(r["ctrl"]["state"]))


def exit_cases():
    rng = np.random.default_rng(42)
    P6 = R.poisson27(6)
    H4 = R.hex_box_csr((4, 3, 3), (0, 0, 0), (4, 3, 3))
    cases = {}
    bP = P6 @ rng.standard_normal(P6.shape[0])
    # converged at the first verification
    cases["converge_first_verify"] = case(P6, bP, minv=1.0 / P6.diagonal(), tol=1e-8, maxiter=200, margin=True,
                                          path=lambda rs: kinds(rs).count(VERIFY) == 1 and _stop(rs)[:2] == (VERIFY, 0))
    # TooSmallTolerance: the recurrence goes below tol*||b||, the true residual cannot.  MaxMSteps = min(nglob/50, 5,
    # nglob - maxiter) with each term the smallest in turn: 3 (nglob/50 < 5), 5, 1, 2, 0 and negative.  The loop stops at the
    # verification where MoreSteps reaches MaxMSteps (the first one when MaxMSteps <= 1), every verification before it failed.
    for tag, ng, mi, mm in [("nglob50_lt5", 150, 100, 3), ("nglob50_eq5", 300, 100, 5), ("ngmi_1", 401, 400, 1),
                            ("ngmi_2", 402, 400, 2), ("ngmi_0", 400, 400, 0), ("ngmi_neg", 300, 400, -100)]:
        assert min(ng // 50, 5, ng - mi) == mm
        cases[f"too_small_{tag}"] = case(P6, bP, minv=1.0 / P6.diagonal(), tol=1e-19, maxiter=mi, n_global=ng, too_small=True,
                                         max_stag=10,
                                         path=lambda rs, mm=mm: _stop(rs)[:2] == (VERIFY, 3) and
                                         int(_stop_rec(rs)["ctrl"]["moresteps"]) == max(mm, 1) and
                                         kinds(rs).count(VERIFY) == max(mm, 1))
    # stagnation: x0 = 2^50 with A x0 exact and b off by 3 ulps in five entries: every step is a few ulps of five
    # entries of x, while eps*||x|| spans sqrt(10^4) = 100 entries (a margin of ~100).  Flag 3 comes from the host
    # verification path: the trigger fires on stag >= max_stag before the dead branch at the end of ctrl_norms.
    n = 10000
    d = 1.0 + (np.arange(n) % 7) / 8.0
    x0 = np.full(n, 2.0 ** 50)
    bs = d * x0
    for j in (11, 2000, 5003, 7777, 9001):
        bs[j] += 3 * np.spacing(bs[j])
    for ms in (1, 2, 3, 0):
        cases[f"stag_max{ms}"] = case(_diag(d), bs, x0=x0, tol=1e-30, maxiter=60, n_global=BIG, max_stag=ms, margin=True,
                                      too_small=False,
                                      path=lambda rs, ms=ms: _stop(rs)[:2] == (VERIFY, 3) and
                                      int(_stop_rec(rs)["ctrl"]["stag"]) >= (ms if ms > 0 else 3) and
                                      int(_stop_rec(rs)["ctrl"]["moresteps"]) < 5 and not any(
                                          int(r["kind"]) == ITER and int(r["ctrl"]["flag"]) == 3 for r in rs))
    # alpha = rho/pq underflows to 0 while x = 0: the stagnation test compares 0 < 0, which is false (`<=` would count a
    # stagnating step and, with max_stag = 1, trigger a verification); the loop runs to maxiter with stag 0
    cases["stag_test_at_equality"] = case(_diag([1e30]), [3e-162], minv=[1e300], tol=1e-30, maxiter=1, n_global=BIG, max_stag=1,
                                          margin=True, too_small=False,
                                          path=lambda rs: float(rs[1]["ctrl"]["alpha"]) == 0.0 and VERIFY not in kinds(rs) and
                                          all(int(r["ctrl"]["stag"]) == 0 for r in rs) and _stop(rs)[2] == ST_EXHAUSTED)
    # flag 2 at iteration 0 (k_rz) and at iteration 1 (#inf(z) of k_update): Minv finite, z = Minv r overflows later
    m2 = np.ones(50)
    m2[3] = np.inf
    D50 = _diag(np.linspace(1, 2, 50))
    b50 = rng.standard_normal(50)
    cases["flag2_iter0"] = case(D50, b50, minv=m2, margin=True, path=lambda rs: _stop(rs)[:2] == (HEAD, 2))
    T = sp.diags([np.full(49, -0.5), np.full(50, 2.0), np.full(49, -0.5)], [-1, 0, 1]).tocsr()
    bt = 1e6 * rng.standard_normal(50)
    bt[10] = 0.0
    mt = np.ones(50)
    mt[10] = 1e308
    cases["flag2_later"] = case(T, bt, minv=mt, margin=True,
                                path=lambda rs: _stop(rs)[:2] == (ITER, 2) and int(rs[0]["ctrl"]["state"]) == 0)
    # flag 4 from each condition
    cases["flag4_rho0_iter0"] = case(D50, b50, minv=np.zeros(50), margin=True, path=lambda rs: _stop(rs)[:2] == (HEAD, 4))
    cases["flag4_rho0_later"] = case(_diag([1.0, 1.0]), [1.0, 1.0], minv=[1.0, 0.0], tol=1e-12, margin=True,
                                     path=lambda rs: _stop(rs)[:2] == (ITER, 4) and float(rs[1]["inp"][RZ]) == 0.0)
    cases["flag4_rho_inf"] = case(_diag([1.0, 1.0]), [1e5, 1.0], minv=[1e300, 1.0], margin=True,
                                  path=lambda rs: _stop(rs)[:2] == (HEAD, 4) and np.isinf(float(rs[0]["inp"][RZ])))
    cases["flag4_beta0"] = case(_diag([1.0, 1.0]), [1e100, 1.0], minv=[1.0, 1e-200], tol=1e-200, margin=True,
                                path=lambda rs: _stop(rs)[:2] == (ITER, 4) and float(rs[1]["ctrl"]["rho"]) == 1e-200)
    cases["flag4_pq0"] = case(_diag([0.0, 0.0]) + sp.csr_matrix((2, 2)), [1.0, 2.0], margin=True,
                              path=lambda rs: _stop(rs)[:2] == (ITER, 4) and float(rs[1]["inp"][PQ]) == 0.0)
    cases["flag4_pq_neg"] = case(_diag(np.concatenate([np.ones(25), -np.ones(25)])), b50, tol=1e-10, margin=True,
                                 path=lambda rs: _stop(rs)[:2] == (ITER, 4) and float(_stop_rec(rs)["inp"][PQ]) < 0)
    cases["flag4_pq_inf"] = case(_diag([1e300]), [1e10], margin=True,
                                 path=lambda rs: _stop(rs)[:2] == (ITER, 4) and np.isinf(float(rs[1]["inp"][PQ])))
    cases["flag4_alpha_inf"] = case(_diag([1e-310]), [1.0], margin=True,
                                    path=lambda rs: _stop(rs)[:2] == (ITER, 4) and 0 < float(rs[1]["inp"][PQ]) < 1e-300)
    # maxiter 1; NaN in Minv (runs to maxiter, flag 1)
    cases["maxiter1"] = case(P6, bP, minv=1.0 / P6.diagonal(), tol=1e-12, maxiter=1, margin=True,
                             path=lambda rs: kinds(rs) == [HEAD, ITER, FINAL] and _stop(rs)[2] == ST_EXHAUSTED)
    mn = 1.0 / P6.diagonal()
    mn[7] = np.nan
    cases["minv_nan"] = case(P6, bP, minv=mn, tol=1e-8, maxiter=15, margin=True,
                             path=lambda rs: _stop(rs)[2] == ST_EXHAUSTED and np.isnan(float(rs[0]["ctrl"]["rho"])))
    # flag 1 on a problem whose residual grows first (XMin still aliased) and later (XMin frozen)
    bh = rng.standard_normal(H4.shape[0])
    for mi in (1, 2, 3, 6, 12, 30):
        cases[f"flag1_maxiter{mi}"] = case(H4, bh, minv=1.0 / H4.diagonal(), tol=1e-14, maxiter=mi,
                                           path=lambda rs: _stop(rs)[:2] == (ITER, 1) and _stop(rs)[2] == ST_EXHAUSTED)
    # early exits: b = 0, and an initial guess that is already good enough
    x0e = rng.standard_normal(P6.shape[0])
    cases["early_b0"] = case(P6, np.zeros(P6.shape[0]), x0=x0e, margin=True, path=lambda rs: len(rs) == 0)
    cases["early_x0_good"] = case(P6, P6 @ x0e, x0=x0e, tol=1e-6, margin=True, path=lambda rs: len(rs) == 0)
    return cases


def ref_solve(c, trace=None):
    p = R.CsrPart(c["A"], c["b"], x0=c["x0"], w=c["w"])
    return R.ref_pcg([p], [c["minv"]], c["tol"], c["maxiter"], nglob=c["n_global"], exist_dp0=c["minv"] is not None,
                     trace=trace, maxstag=c["max_stag"])
