"""The index-free hex-box operator's host restatement (tests/hexop_cases.py) and its C ABI, without a GPU: the slots the
kernel visits per dof are the ordered operator's slot lists, and its long-double product is the generated matrix's."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import ref_pcg as R
from pcg_mpi_solver_b200 import _lib
from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_type_group
from tests import hexop_cases as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("pcgb_hexop_create", "pcgb_hexop_destroy", "pcgb_hexop_apply", "pcgb_hexop_diag", "pcgb_hexop_bytes",
       "pcgb_solver_create_hexop")


@pytest.mark.parametrize("box", C.BOXES)
def test_enumeration_is_the_ordered_slot_order(box):
    blk = HexBlock(*box)
    grp, eff, ndof = hex_type_group(blk)
    assert C.node_slots(blk) == C.group_slots(grp, eff, ndof)


@pytest.mark.parametrize("box", C.BOXES)
@pytest.mark.parametrize("field", [False, True])
def test_long_double_product_is_the_csr(box, field):
    rng = np.random.default_rng(sum(box[2]) + 7 * field)
    blk = HexBlock(*box, h=0.5, E=3.0, nu=0.45)
    nel = int(np.prod(blk.ne))
    ck = rng.uniform(0.01, 100.0, nel) if field else np.full(nel, blk.E * blk.h)
    x = rng.standard_normal(blk.n)
    rows = np.arange(blk.n)
    y, _, _ = C.ref_rows(blk, rows, lambda i: x[i], lambda e: ck[e])
    if field:
        grp, eff, ndof = hex_type_group(blk, E_field=ck.reshape(tuple(reversed(blk.ne))) / blk.h)
        from tests import ebe_ordered_cases as EC
        want, scale, _ = EC.ref_apply([grp], eff, ndof, x)
    else:
        A = R.hex_box_csr(blk.ng, blk.e0, blk.ne, E=blk.E, nu=blk.nu, h=blk.h)
        want = A @ x
        scale = abs(A) @ np.abs(x)
    assert (np.abs(np.asarray(y, dtype=np.float64) - np.asarray(want, dtype=np.float64)) <= 1e-13 * np.maximum(scale, 1e-300)).all()


def test_abi_declared_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "pcgb200.h")).read()
    for name in NEW:
        assert re.search(rf"\b{name}\(", hdr), name
        assert name in _lib.SIGNATURES, name
    so = _lib.LIB_PATH
    if not os.path.exists(so):
        pytest.skip("library not built")
    syms = subprocess.run(["nm", "-D", "--defined-only", so], stdout=subprocess.PIPE, text=True, check=True).stdout
    for name in NEW:
        assert re.search(rf"\bT {name}$", syms, re.M), name
