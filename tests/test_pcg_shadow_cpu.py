"""CPU pin of the control-logic restatement (tests/pcg_shadow.py) against the reference restatement oracle/ref_pcg.py:
fed ref_pcg's own reduced values step by step, the shadow must make exactly ref_pcg's decisions and reach the
exit path each problem of tests/pcg_cases.py is built for."""
import numpy as np
import pytest

from oracle import ref_pcg as R
from pcg_mpi_solver_b200.solver import TRACE_DTYPE
from tests import pcg_cases as C
from tests import pcg_shadow as S

EXIT = C.exit_cases()


def _existing():
    rng = np.random.default_rng(3)
    P8 = R.poisson27(8)
    H8 = R.hex_box_csr((8, 8, 8), (0, 0, 0), (8, 8, 8))
    P10 = R.poisson27(10)
    return {
        "poisson8_jacobi": C.case(P8, P8 @ rng.standard_normal(P8.shape[0]), minv=1.0 / P8.diagonal(), tol=1e-8, maxiter=1000),
        "hex8_resvec": C.case(H8, rng.standard_normal(H8.shape[0]), minv=1.0 / H8.diagonal(), tol=1e-9, maxiter=5000),
        "poisson10_x0_noprec": C.case(P10, P10 @ rng.standard_normal(P10.shape[0]), x0=rng.standard_normal(P10.shape[0]),
                                      tol=1e-9, maxiter=1000),
        "poisson8_tol16": C.case(P8, P8 @ rng.standard_normal(P8.shape[0]), minv=1.0 / P8.diagonal(), tol=1e-16, maxiter=400),
        "poisson8_weights": C.case(P8, rng.standard_normal(P8.shape[0]), minv=1.0 / P8.diagonal(), tol=1e-10, maxiter=1000,
                                   w=rng.uniform(0.2, 1.0, P8.shape[0])),
    }


def replay_ref(c):
    """(ref result, shadow, shadow records, ref's stag after every norms step) for one case."""
    tr = []
    ref = C.ref_solve(c, trace=tr)
    if len(tr) == 0 or tr[-1]["step"] == "start":      # early exit before the loop: nothing to replay
        return ref, None, np.zeros(0, dtype=TRACE_DTYPE), []
    recs = S.records_from_ref(tr)
    sh = S.replay(recs, c["tol"], c["maxiter"], c["n_global"], c["max_stag"], check_ctrl=False)
    # per-iteration stagnation counter of the reference
    ref_stag = [e["stag"] for e in tr if e["step"] == "norms"]
    return ref, sh, S.to_array(sh), ref_stag


def _check_same_decisions(c, name):
    out = replay_ref(c)
    ref = out[0]
    if out[1] is None:
        assert c["path"] is None or c["path"](out[2]), name
        return
    _, sh, recs, ref_stag = out
    res = sh.result
    assert res is not None, "the replay did not reach the finalisation"
    assert res["flag"] == ref["Flag"], (name, res, ref["Flag"])
    assert res["iters"] == ref["Iter"], (name, res["iters"], ref["Iter"])
    assert S.same_bits(res["relres"], ref["RelRes"]), (name, res["relres"], ref["RelRes"])
    assert res["imin"] == ref["iMin"]
    assert res["stag"] == ref["stag"] and res["moresteps"] == ref["moresteps"]
    assert res["too_small_tol"] == bool(ref["too_small_tol"])
    if c.get("too_small") is not None:
        assert res["too_small_tol"] == c["too_small"], name
    assert (recs[-1]["ctrl"]["alias"] == 1) == bool(ref["aliased"])
    assert sh.stags == ref_stag
    if c["path"] is not None:
        assert c["path"](recs), (name, [int(k) for k in recs["kind"]])


@pytest.mark.parametrize("name", sorted(_existing()))
def test_shadow_makes_ref_decisions_existing_problems(name):
    _check_same_decisions(_existing()[name], name)


@pytest.mark.parametrize("name", sorted(EXIT))
def test_shadow_makes_ref_decisions_exit_paths(name):
    _check_same_decisions(EXIT[name], name)


def test_max_msteps_terms():
    assert S.max_msteps(100, 10) == 2          # nglob/50 < 5
    assert S.max_msteps(250, 10) == 5          # 5
    assert S.max_msteps(1000, 999) == 1        # nglob - maxiter = 1
    assert S.max_msteps(1000, 998) == 2
    assert S.max_msteps(1000, 1000) == 0 and S.max_msteps(100, 300) == -200


def test_shadow_flags_a_wrong_record():
    """The replay is strict: one changed bit of one field of one record fails it."""
    c = _existing()["poisson8_jacobi"]
    tr = []
    C.ref_solve(c, trace=tr)
    recs = S.records_from_ref(tr)
    good = S.to_array(S.replay(recs, c["tol"], c["maxiter"], c["n_global"], check_ctrl=False))
    S.replay(good, c["tol"], c["maxiter"], c["n_global"])       # its own records replay cleanly
    for field, k in (("rho_prev", 3), ("stag", 5), ("moresteps", len(good) - 2)):
        bad = good.copy()
        if field in S.FLOAT_FIELDS:
            bad[k]["ctrl"][field] = np.nextafter(bad[k]["ctrl"][field], np.inf)
        else:
            bad[k]["ctrl"][field] += 1
        with pytest.raises(AssertionError):
            S.replay(bad, c["tol"], c["maxiter"], c["n_global"])
