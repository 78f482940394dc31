"""The coloured matrix-free operator (EbeMatrixColored, csrc/ebe_color.cuh) bit for bit against its colour-order
restatement (tests/ebe_color_cases.py::color_f64) at the kernel edges: every pattern size, block tail and sign mode of
the synthetic groups, the device-assembly cases (repeated dofs in one element, in one 32-lane pass and across passes;
patterns that are not node-major; 300 groups; empty groups; no free dof), hex boxes, concrete, the warp-kernel fallback
when every constant-memory slot is taken, caller colourings and the colour-order pin.  Also: the launch count, refusals
that leave nothing behind, and the atomic EbeMatrix entrywise on the same cases."""
import ctypes
import gc
import os

import numpy as np
import pytest

from tests import asm_cases as A
from tests import ebe_color_cases as C
from tests.test_gpu_ebe import SIGNS, _assert_entrywise, _colored_launches, _synthetic_groups

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _asm_subs():
    subs = [(f"pattern_{nd}_{v}", A.pattern_case(nd, v)) for nd in A.PATTERN_SIZES if nd <= 96 for v in A.PATTERN_VARIANTS]
    subs += [("structure", A.structure_case()), ("duplicate", A.duplicate_case()), ("many_groups", A.many_groups_case()),
             ("spd", A.spd_case()), ("order", A.order_case()), ("no_rows", A.no_rows_case())]
    return subs


ASM = [name for name, _ in _asm_subs()]


def _asm(name):
    sub = dict(_asm_subs())[name]
    return C.near_symmetric(sub.groups), sub.loc_dof_eff, sub.ndof


def _apply_bits(op, x, cuda):
    """op.apply_local(x) into a NaN-filled output, as float64 on the host."""
    import torch
    out = torch.full((op.shape[0],), float("nan"), dtype=torch.float64, device=cuda)
    op.apply_local(torch.from_numpy(np.ascontiguousarray(x)).to(cuda), out=out)
    return out.cpu().numpy()


def _colours_of(groups, ndof):
    from pcg_mpi_solver_b200.coloring import color_groups
    return color_groups(groups, ndof)[0]


def _assert_bits(y, want, what=""):
    assert not np.isnan(y).any(), f"{what}: {int(np.isnan(y).sum())} entries never written"
    bad = np.nonzero(y.view(np.int64) != np.asarray(want, dtype=np.float64).view(np.int64))[0]
    assert bad.size == 0, f"{what}: {bad.size} of {y.size} entries differ, first {bad[:5]}: {y[bad[:5]]} vs {want[bad[:5]]}"


def _check(cuda, groups, eff, ndof, x, colours=None, what=""):
    """Build the operator (computed colouring, or `colours`), compare one application with color_f64 bit for bit and a
    second application with the first.  Returns the operator and y."""
    from pcg_mpi_solver_b200.ebe import EbeMatrixColored
    E = EbeMatrixColored(groups, eff, ndof, device=cuda, colors_per_group=colours)
    cols = colours if colours is not None else _colours_of(groups, ndof)
    y = _apply_bits(E, x, cuda)
    _assert_bits(y, C.color_f64(groups, cols, eff, ndof, x), what)
    _assert_bits(_apply_bits(E, x, cuda), y, what + " (again)")
    return E, y


def _expected_launches(groups, colours, slotted=True):
    """(colour, 24-dof group) pairs with elements when the 24-dof patterns hold constant-memory slots, plus one per colour
    with a non-empty warp-kernel slice; with no slot, one per colour with elements."""
    n = 0
    ncol = max([int(c.max()) + 1 for c in colours if c.size], default=0)
    for c in range(ncol):
        nds = [g.loc_dof.shape[0] for g, col in zip(groups, colours) if (col == c).any()]
        if slotted:
            n += sum(nd == 24 for nd in nds) + int(any(nd != 24 for nd in nds))
        else:
            n += int(bool(nds))
    return n


@pytest.mark.parametrize("signs", list(SIGNS))
def test_colored_synthetic_groups_bit_for_bit(cuda, signs):
    """nd 1..96 x ne 0..129 (block tails of both kernels) and one 3000-element 24-dof group, in all three sign modes."""
    rng = np.random.default_rng(40 + list(SIGNS).index(signs))
    groups, eff, ndof = _synthetic_groups(rng, SIGNS[signs])
    gc.collect()
    x = rng.standard_normal(len(eff))
    _check(cuda, groups, eff, ndof, x, what=signs)


@pytest.mark.parametrize("name", ASM)
def test_colored_asm_cases_bit_for_bit(cuda, name):
    """Every device-assembly case with patterns up to 96, Ke symmetric to a few ulps but not bit for bit: repeated dofs
    (duplicate), patterns that are not node-major (spd, order, many_groups), empty groups (structure), n = 0 (no_rows)."""
    groups, eff, ndof = _asm(name)
    gc.collect()
    x = np.random.default_rng(len(name)).standard_normal(len(eff)) * 10.0 ** np.random.default_rng(1).uniform(-2, 2, len(eff))
    E, _ = _check(cuda, groups, eff, ndof, x, what=name)
    assert E.launches() == _expected_launches(groups, _colours_of(groups, ndof))


def test_colored_duplicate_case_repeats(cuda):
    """duplicate_case one pass (local 3 and 10), two passes (5 and 38) and three times (1, 2, 33), element by element:
    a single element of each kind, so that every dof's sum is that element's rows in ascending local index."""
    groups, eff, ndof = _asm("duplicate")
    g = groups[0]
    for lo, hi in ((0, 20), (20, 40), (40, 50), (50, 60)):
        for e in (lo, hi - 1):
            one = [type(g)(0, g.loc_dof[:, e:e + 1], g.sign[:, e:e + 1], g.ck[e:e + 1], g.ke, np.arange(1))]
            x = np.random.default_rng(e).standard_normal(len(eff))
            _check(cuda, one, eff, ndof, x, colours=[np.zeros(1, np.int64)], what=f"element {e}")


def test_colored_hex_boxes_and_partitions(cuda, tmp_path):
    """A clamped hex box, interior boxes of a 2 x 2 x 1 cut, and the subdomains of a 3-way METIS partition of a hex
    model (signs-free 24-dof groups on the thread kernel)."""
    from oracle.hex_mdf import write_hex_mdf
    from pcg_mpi_solver_b200.hexmesh import HexBlock, block_grid, hex_type_group, partition_blocks
    from pcg_mpi_solver_b200.model import load_mdf
    from pcg_mpi_solver_b200.partition import partition_mesh
    rng = np.random.default_rng(50)
    cases = [hex_type_group(HexBlock((9, 7, 5), (0, 0, 0), (9, 7, 5), h=1.0 / 9))]
    for blk in partition_blocks((8, 6, 4), block_grid(4)):
        blk.h = 1.0 / 8
        cases.append(hex_type_group(blk))
    write_hex_mdf(str(tmp_path), (8, 6, 5))
    for sub in partition_mesh(load_mdf(str(tmp_path)), 3, assemble=False):
        cases.append((sub.groups, sub.loc_dof_eff, sub.ndof))
    for k, (groups, eff, ndof) in enumerate(cases):
        groups = groups if isinstance(groups, list) else [groups]
        x = rng.standard_normal(len(eff))
        E, _ = _check(cuda, groups, eff, ndof, x, what=f"hex case {k}")
        assert E.launches() == _expected_launches(groups, _colours_of(groups, ndof))


def test_colored_concrete(cuda):
    zp = os.path.join(ROOT, "oracle", "_ref", "concrete.zip")
    if not os.path.exists(zp):
        pytest.skip("concrete.zip not staged")
    from pcg_mpi_solver_b200.partition import partition_mesh
    sub = partition_mesh(zp, 1, assemble=False)[0]
    x = np.random.default_rng(51).standard_normal(sub.n)
    gc.collect()
    _check(cuda, sub.groups, sub.loc_dof_eff, sub.ndof, x, what="concrete")


@pytest.mark.parametrize("name", ["spd", "hex"])
def test_colored_slot_fallback_same_bits_fewer_launches(cuda, name):
    """With every constant-memory slot taken, the 24-dof groups run on the warp kernel: the same bits, one launch per
    colour (fewer than slotted when a colour also has warp-kernel groups)."""
    from pcg_mpi_solver_b200.ebe import EbeMatrix
    from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_type_group
    if name == "spd":
        groups, eff, ndof = _asm("spd")
    else:
        g, eff, ndof = hex_type_group(HexBlock((7, 6, 5), (0, 0, 0), (7, 6, 5), h=1.0 / 7))
        groups = [g]
    colours = _colours_of(groups, ndof)
    rng = np.random.default_rng(52)
    x = rng.standard_normal(len(eff))
    gc.collect()
    E, y = _check(cuda, groups, eff, ndof, x, what=name)
    slotted = E.launches()
    assert slotted == _expected_launches(groups, colours)
    del E
    gc.collect()
    fill, fe, fn = _synthetic_groups(rng, 0.2, shapes=[(24, 129)] * 10)      # nine distinct Ke fill the table
    held = EbeMatrix(fill, fe, fn, device=cuda)
    assert _colored_launches(cuda, rng) == 1
    F, yf = _check(cuda, groups, eff, ndof, x, what=name + " on the warp kernel")
    _assert_bits(yf, y, name + " fallback vs slotted")
    assert F.launches() == _expected_launches(groups, colours, slotted=False) <= slotted
    if name == "spd":                                   # its colours mix the 24-dof group with warp-kernel groups
        assert F.launches() < slotted
    del F, held
    gc.collect()


def test_colored_caller_colourings(cuda):
    """hex_parity_colors on a hex box (8 colours) and the colour-order pin (only the documented colour order gives its
    vector)."""
    from pcg_mpi_solver_b200.coloring import hex_parity_colors
    from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_type_group
    nx, ny, nz = 7, 5, 4
    g, eff, ndof = hex_type_group(HexBlock((nx, ny, nz), (0, 0, 0), (nx, ny, nz), h=1.0 / nx))
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    pc, pn = hex_parity_colors(ex.ravel(), ey.ravel(), ez.ravel())
    x = np.random.default_rng(53).standard_normal(len(eff))
    E, _ = _check(cuda, [g], eff, ndof, x, colours=[pc], what="parity")
    assert E.ncolors == pn and E.launches() == pn
    groups, colours, eff, ndof, x, want, rev = C.colour_order_pin()
    E, y = _check(cuda, groups, eff, ndof, x, colours=colours, what="order pin")
    _assert_bits(y, want, "order pin")
    assert not np.array_equal(y, rev)


def test_colored_refusals_leave_nothing_behind(cuda):
    """A shared-dof colouring and a non-symmetric Ke are refused with no device memory and no constant-memory slot taken;
    pcgb_ebe2_create with phases out of order returns PCGB_ERR_ARG and no handle."""
    import dataclasses

    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.ebe import EbeMatrixColored
    rng = np.random.default_rng(54)
    gc.collect()
    assert _colored_launches(cuda, rng) == 2
    groups, eff, ndof = _asm("spd")
    before = torch.cuda.memory_allocated(cuda)
    with pytest.raises(ValueError):
        EbeMatrixColored(groups, eff, ndof, device=cuda, colors_per_group=C.old_colouring(groups, ndof))
    skew = [dataclasses.replace(g, ke=g.ke + np.triu(np.ones_like(g.ke), 1)) for g in groups]
    with pytest.raises(ValueError):
        EbeMatrixColored(skew, eff, ndof, device=cuda)
    gc.collect()
    assert torch.cuda.memory_allocated(cuda) == before
    assert _colored_launches(cuda, rng) == 2
    keep = []
    cg = (_lib.EbeGroup * 2)()
    for k in range(2):
        ke = rng.standard_normal((24, 24))
        ke = ke + ke.T
        d_idx = torch.arange(24 * k, 24 * k + 24, dtype=torch.int32, device=cuda)
        d_ck = torch.ones(1, dtype=torch.float64, device=cuda)
        keep += [ke, d_idx, d_ck]
        cg[k].nd, cg[k].ne, cg[k].d_idx, cg[k].d_ck, cg[k].d_sign, cg[k].ke_host = 24, 1, d_idx.data_ptr(), d_ck.data_ptr(), None, ke.ctypes.data
    phase = (ctypes.c_int32 * 2)(1, 0)
    h = ctypes.c_void_p()
    with torch.cuda.device(cuda):
        assert _lib.load().pcgb_ebe2_create(48, 2, cg, phase, ctypes.byref(h)) == -1    # PCGB_ERR_ARG
    assert not h
    assert _colored_launches(cuda, rng) == 2


@pytest.mark.parametrize("name", [n for n in ASM if n != "no_rows"])
def test_atomic_ebe_asm_cases_entrywise(cuda, name):
    """The atomic EbeMatrix on the same cases (repeated dofs on its warp kernel among them) against the long-double
    reference, entrywise."""
    from pcg_mpi_solver_b200.ebe import EbeMatrix
    groups, eff, ndof = _asm(name)
    gc.collect()
    x = np.random.default_rng(len(name) + 7).standard_normal(len(eff))
    E = EbeMatrix(groups, eff, ndof, device=cuda)
    y = _apply_bits(E, x, cuda)
    assert not np.isnan(y).any()
    _assert_entrywise(y, groups, eff, ndof, x)
