"""CPU checks of the ordered matrix-free operator: its C entry points load and refuse to run without a device, the
long-double restatement the GPU tests use agrees with the oracle's EBE apply, and the order-pin case cancels."""
import ctypes

import numpy as np
import pytest

from tests import asm_cases as AC
from tests import ebe_ordered_cases as C

SYMBOLS = ("pcgb_ebe_ordered_create", "pcgb_ebe_ordered_destroy", "pcgb_ebe_ordered_apply", "pcgb_ebe_ordered_bytes",
           "pcgb_solver_create_ebe_ordered")


def test_symbols_load_and_need_a_device():
    import torch
    from pcg_mpi_solver_b200 import _lib
    lib = _lib.load()
    for name in SYMBOLS:
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = ctypes.c_void_p()
    assert lib.pcgb_ebe_ordered_create(0, 0, None, ctypes.byref(h)) == -4 and not h
    assert b"no CPU fallback" in lib.pcgb_last_error()
    fake = ctypes.c_void_p(1)           # never dereferenced: the device check comes first
    assert lib.pcgb_solver_create_ebe_ordered(fake, None, None, ctypes.byref(h)) == -4 and not h
    assert lib.pcgb_ebe_ordered_apply(None, None, None, None) == -1
    assert lib.pcgb_ebe_ordered_destroy(None) == 0 and lib.pcgb_ebe_ordered_bytes(None) == 0
    # argument refusals come before the device check
    assert lib.pcgb_ebe_ordered_create(2**30, 0, None, ctypes.byref(h)) == -1


def _oracle_apply(sub, x):
    from oracle import ref_pcg as R
    part = R.EbePart(sub.to_refmeshpart())
    xf = np.zeros(sub.ndof)
    xf[sub.loc_dof_eff] = x
    return part.matvec_full(xf)[sub.loc_dof_eff]


@pytest.mark.parametrize("case", ["pattern", "structure", "duplicate", "many_groups", "spd"])
def test_restatement_matches_oracle_ebe_apply(case):
    sub = {"pattern": lambda: AC.pattern_case(33, "signs20"), "structure": AC.structure_case, "duplicate": AC.duplicate_case,
           "many_groups": AC.many_groups_case, "spd": AC.spd_case}[case]()
    x = np.random.default_rng(2).standard_normal(sub.n)
    y, b, k = C.ref_apply(sub.groups, sub.loc_dof_eff, sub.ndof, x)
    yo = _oracle_apply(sub, x)
    assert (np.abs(yo - y) <= (k + 2) * C.EPS * b).all()
    yf = C.ordered_f64(sub.groups, sub.loc_dof_eff, sub.ndof, x) if case != "many_groups" else None
    if yf is not None:
        assert (np.abs(yf - y) <= (k + 2) * C.EPS * b).all()


def test_order_pin_reaches_its_cancellation():
    groups, eff, ndof, x, want = C.order_pin()
    y, b, k = C.ref_apply(groups, eff, ndof, x)
    assert (y == 1.0).all()                                        # exact value: every 1 survives in long double
    assert np.array_equal(C.ordered_f64(groups, eff, ndof, x), want)
    elem = C.ordered_f64(groups, eff, ndof, x, order="element")
    assert not np.array_equal(elem, want)
    # every reversal of a dof's list changes which slot comes last: the result differs
    vals = C.slot_values(groups, eff, ndof, x)
    rev = np.zeros(3)
    for dof, _, v, *_ in sorted(vals, key=lambda t: -t[1]):
        rev[dof] = rev[dof] + v
    assert not np.array_equal(rev, want)
