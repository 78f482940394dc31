"""Host restatement of the PCG control logic, in plain Python floats, for replaying a loop trace bit for bit.

It restates `ctrl_alpha`, `ctrl_head`, `ctrl_next` and `ctrl_norms` (csrc/pcg_kernels.cuh), the host verification
branch, MaxMSteps and the finalisation choice of `solve_on` (csrc/pcgb_api.cu).  Fed the reduced values a solve
consumed (the records of `SubdomainOperator.solve(trace=...)`), it must reproduce the control block after every step
exactly, and then the result of the solve.  Because it uses the device's own sums, its decisions do not depend on
rounding: a wrong weight, a stale rho, an off-by-one in MaxMSteps change a field of some record.

IEEE division and sqrt are correctly rounded in Python as on the device.  The one expression nvcc may contract is the
stagnation test `normp*|alpha| < eps*normx` (eps*normx is exact: eps is a power of two), so the product is evaluated
both rounded and exact; where the two disagree either is accepted (the device's record decides) and the case is counted.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

EPS = 2.220446049250313e-16
ST_RUN, ST_TRIGGER, ST_BREAK, ST_EXHAUSTED = 0, 1, 2, 3
HEAD, ITER, VERIFY, RESUME, FINAL = 0, 1, 2, 3, 4
PQ, PP, XX, RR, RZ, NINF, BB, R0R0 = range(8)
FLOAT_FIELDS = ("rho", "rho_prev", "alpha", "beta", "pq", "normr", "normp", "normx", "normr_act", "normrmin", "tolb", "n2b", "eps")
INT_FIELDS = ("state", "flag", "iter", "stag", "moresteps", "imin", "xcur", "xmin", "maxiter", "maxstag", "fixed_iters", "alias")


def c_div(a: float, b: float) -> float:
    """a / b with IEEE semantics (Python raises on b == 0)."""
    try:
        return a / b
    except ZeroDivisionError:
        if math.isnan(a) or a == 0.0:
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)


def c_sqrt(a: float) -> float:
    return math.nan if (math.isnan(a) or a < 0.0) else math.sqrt(a)


def same_bits(a: float, b: float) -> bool:
    """Bit equality of two doubles (any NaN equals any NaN: payloads are not part of the arithmetic)."""
    a, b = float(a), float(b)
    if math.isnan(a) and math.isnan(b):
        return True
    return struct.pack("<d", a) == struct.pack("<d", b)


def max_msteps(nglob: int, maxiter: int) -> int:
    """MaxMSteps = min(nglob/50, 5, nglob - maxiter) (pcg_solver.py:404, integer division of positive numbers)."""
    mm = min(int(nglob) // 50, 5)
    return min(mm, int(nglob) - int(maxiter))


# stagnation tests evaluated, and those where the rounded and the exact product decided differently (all replays of a run)
FMA_STATS = {"tests": 0, "disagreements": 0}


class Shadow:
    def __init__(self, tol, maxiter, n_global, max_stag=3, fixed_iters=False):
        self.tol, self.maxiter, self.nglob = float(tol), int(maxiter), int(n_global)
        self.maxstag = int(max_stag) if max_stag > 0 else 3
        self.fixed = 1 if fixed_iters else 0
        self.maxmsteps = max_msteps(self.nglob, self.maxiter)
        self.c = None
        self.fma_disagreements = 0   # stagnation tests where the rounded and the exact product decide differently
        self.result = None
        self.resvec = {}
        self.stags = []              # stag after every norms step
        self.records = []            # (kind, inputs, control block after the step) of every replayed record

    # ---- set-up of solve_on before the loop
    def start(self, bb, r0r0):
        n2b, normr = c_sqrt(bb), c_sqrt(r0r0)
        self.c = dict(rho=1.0, rho_prev=1.0, alpha=0.0, beta=0.0, pq=0.0, normr=normr, normp=0.0, normx=0.0, normr_act=normr,
                      normrmin=normr, tolb=self.tol * n2b, n2b=n2b, eps=EPS, state=ST_RUN, flag=1, iter=0, stag=0, moresteps=0,
                      imin=0, xcur=0, xmin=0, maxiter=self.maxiter, maxstag=self.maxstag, fixed_iters=self.fixed, alias=1)

    # ---- device control logic
    def alpha(self, pq):
        c = self.c
        c["pq"] = pq
        if pq <= 0.0 or math.isinf(pq):
            c["flag"], c["state"] = 4, ST_BREAK
            return
        a = c_div(c["rho"], pq)
        if math.isinf(a):
            c["flag"], c["state"] = 4, ST_BREAK
            return
        c["alpha"] = a

    def head(self, rz, ninf):
        c = self.c
        if ninf > 0.0:
            c["flag"], c["state"] = 2, ST_BREAK
            return
        c["rho_prev"] = c["rho"]
        c["rho"] = rz
        if rz == 0.0 or math.isinf(rz):
            c["flag"], c["state"] = 4, ST_BREAK
            return
        if c["iter"] > 0:
            beta = c_div(rz, c["rho_prev"])
            if beta == 0.0 or math.isinf(beta):
                c["flag"], c["state"] = 4, ST_BREAK
                return
            c["beta"] = beta

    def next(self, rz, ninf):
        c = self.c
        if c["iter"] + 1 >= c["maxiter"]:
            c["state"] = ST_EXHAUSTED
            return
        c["iter"] += 1
        self.head(rz, ninf)

    def stagnating(self, normp, alpha, normx, device_stag=None):
        lhs_r = normp * abs(alpha)
        rhs = EPS * normx
        plain = lhs_r < rhs
        FMA_STATS["tests"] += 1
        try:
            fused = Fraction(normp) * Fraction(abs(alpha)) < Fraction(rhs)
        except (ValueError, OverflowError):   # inf / nan: no rounding question
            fused = plain
        if plain == fused:
            return plain
        self.fma_disagreements += 1
        FMA_STATS["disagreements"] += 1
        if device_stag is None:
            return plain
        return device_stag == self.c["stag"] + 1

    def norms(self, pp, xx, rr, rz, ninf, device_stag=None):
        c = self.c
        if not c["alias"] and c["xcur"] == c["xmin"]:
            c["xcur"] ^= 1
        normp, normx, normr = c_sqrt(pp), c_sqrt(xx), c_sqrt(rr)
        c["normp"], c["normx"], c["normr"] = normp, normx, normr
        if self.stagnating(normp, c["alpha"], normx, device_stag):
            c["stag"] += 1
        else:
            c["stag"] = 0
        self.stags.append(c["stag"])
        c["normr_act"] = normr
        self.resvec[c["iter"] + 1] = normr
        if not c["fixed_iters"] and (normr <= c["tolb"] or c["stag"] >= c["maxstag"] or c["moresteps"] > 0):
            c["state"] = ST_TRIGGER
            return
        if normr < c["normrmin"]:
            c["normrmin"], c["xmin"], c["imin"], c["alias"] = normr, c["xcur"], c["iter"], 0
        if not c["fixed_iters"] and c["stag"] >= c["maxstag"]:   # unreachable: the trigger above fires first
            c["flag"], c["state"] = 3, ST_BREAK
            return
        self.next(rz, ninf)

    # ---- host side of solve_on
    def verify(self, rr):
        """Verification with the true residual (pcg_solver.py:527-562).  Returns True when the loop stops."""
        c = self.c
        normr_act = c_sqrt(rr)
        c["normr_act"] = normr_act
        self.too_small = False
        if normr_act <= c["tolb"]:
            c["flag"] = 0
            return True
        if c["stag"] >= self.maxstag and c["moresteps"] == 0:
            c["stag"] = 0
        c["moresteps"] += 1
        if c["moresteps"] >= self.maxmsteps:
            self.too_small = True
            c["flag"] = 3
            return True
        if normr_act < c["normrmin"]:
            c["normrmin"], c["xmin"], c["imin"], c["alias"] = normr_act, c["xcur"], c["iter"], 0
        if c["stag"] >= self.maxstag:
            c["flag"] = 3
            return True
        c["state"] = ST_RUN
        return False

    def finalise(self, rr_min):
        c = self.c
        i = c["iter"]
        if c["flag"] == 0:
            relres, it, xout = c_div(c["normr_act"], c["n2b"]), i, c["xcur"]
        else:
            normr_min = c_sqrt(rr_min)
            if normr_min < c["normr_act"]:
                it, relres = c["imin"], c_div(normr_min, c["n2b"])
            else:
                it, relres = i, c_div(c["normr_act"], c["n2b"])
            xout = c["xmin"]
        self.result = dict(flag=c["flag"], iters=it + 1, relres=relres, imin=c["imin"], stag=c["stag"], moresteps=c["moresteps"],
                           too_small_tol=bool(getattr(self, "too_small", False)), xout=xout)
        return self.result


def _ctrl_of(rec):
    c = rec["ctrl"]
    return {f: (float(c[f]) if f in FLOAT_FIELDS else int(c[f])) for f in FLOAT_FIELDS + INT_FIELDS}


def diff_ctrl(mine: dict, dev: dict):
    bad = [f for f in FLOAT_FIELDS if not same_bits(mine[f], dev[f])]
    bad += [f for f in INT_FIELDS if mine[f] != dev[f]]
    return {f: (mine[f], dev[f]) for f in bad}


def replay(records, tol, maxiter, n_global, max_stag=3, fixed_iters=False, check_ctrl=True):
    """Replay a trace.  records: sequence of mappings with 'kind', 'inp' (8 slots) and, when check_ctrl, 'ctrl' (a PcgCtrl
    record).  Every control block must match bit for bit; returns the Shadow (its .result is the solve's outcome)."""
    sh = Shadow(tol, maxiter, n_global, max_stag, fixed_iters)
    for k, rec in enumerate(records):
        kind, v = int(rec["kind"]), [float(a) for a in rec["inp"]]
        dev = _ctrl_of(rec) if check_ctrl else None
        if kind == HEAD:
            assert k == 0, "the iteration-0 head must be the first record"
            sh.start(v[BB], v[R0R0])
            sh.head(v[RZ], v[NINF])
        elif kind == ITER:
            assert sh.c["state"] == ST_RUN, f"record {k}: an iteration ran after the loop stopped"
            sh.alpha(v[PQ])
            if sh.c["state"] == ST_RUN:
                sh.norms(v[PP], v[XX], v[RR], v[RZ], v[NINF], dev["stag"] if dev else None)
        elif kind == VERIFY:
            assert sh.c["state"] == ST_TRIGGER, f"record {k}: verification without a trigger"
            sh.verify(v[RR])
        elif kind == RESUME:
            assert sh.c["state"] == ST_RUN, f"record {k}: head after a verification that stopped the loop"
            sh.next(v[RZ], v[NINF])
        elif kind == FINAL:
            assert k == len(records) - 1, "the finalisation must be the last record"
            if sh.c["state"] == ST_RUN:
                raise AssertionError(f"record {k}: finalisation while the loop still runs")
            sh.finalise(v[RR])
        else:
            raise AssertionError(f"record {k}: unknown kind {kind}")
        if dev is not None:
            d = diff_ctrl(sh.c, dev)
            assert not d, f"record {k} (kind {kind}, iter {dev['iter']}): shadow != device {d}"
        sh.records.append((kind, v, dict(sh.c)))
    return sh


def to_array(sh):
    """The shadow's own records (inputs and its control block after each step) in the device's record layout."""
    import numpy as np
    from pcg_mpi_solver_b200.solver import TRACE_DTYPE
    out = np.zeros(len(sh.records), dtype=TRACE_DTYPE)
    for k, (kind, v, c) in enumerate(sh.records):
        out[k]["kind"] = kind
        out[k]["inp"] = v
        out[k]["local"] = v
        for f, val in c.items():
            out[k]["ctrl"][f] = val
    return out


def records_from_ref(trace):
    """Turn the per-step trace of oracle.ref_pcg.ref_pcg into the record sequence the device writes (kind, inp), so that
    the same Shadow replays the reference's own scalars.  The device consumes the head of iteration i+1 inside the
    record of iteration i (or in a RESUME record after a failed verification)."""
    recs = []

    def rec(kind, **slots):
        inp = [0.0] * 8
        for name, val in slots.items():
            inp[("pq", "pp", "xx", "rr", "rz", "ninf", "bb", "r0r0").index(name)] = float(val)
        recs.append({"kind": kind, "inp": inp})

    ev = list(trace)
    start = ev[0]
    assert start["step"] == "start"
    heads = {e["i"]: e for e in ev if e["step"] == "head"}

    def head_vals(i):
        h = heads.get(i)
        if h is None:
            return dict(rz=0.0, ninf=0.0)
        return dict(rz=h.get("rz", 0.0), ninf=h["ninf"])

    rec(HEAD, bb=start["bb"], r0r0=start["r0r0"], **head_vals(0))
    for k, e in enumerate(ev):
        if e["step"] == "pq":
            nxt = ev[k + 1] if k + 1 < len(ev) else None
            if nxt is None or nxt["step"] != "norms":
                rec(ITER, pq=e["pq"])
                continue
            verified = k + 2 < len(ev) and ev[k + 2]["step"] == "verify"
            hv = dict(rz=0.0, ninf=0.0) if verified else head_vals(e["i"] + 1)
            rec(ITER, pq=e["pq"], pp=nxt["pp"], xx=nxt["xx"], rr=nxt["rr"], **hv)
        elif e["step"] == "verify":
            rec(VERIFY, rr=e["rr"])
            if not e["stop"]:
                rec(RESUME, **head_vals(e["i"] + 1))
        elif e["step"] == "final":
            rec(FINAL, rr=e["rr"])
    return recs
