"""The host restatements of the coloured EBE operator (tests/ebe_color_cases.py) and its colouring, on the CPU: the C helper
against exact rational arithmetic, the orders it must tell apart, the colouring on every pattern layout, and the
refusals EbeMatrixColored makes before it reaches the library."""
import dataclasses

import numpy as np
import pytest

from tests import asm_cases as A
from tests import ebe_color_cases as C


def _small_cases():
    """(name, groups, eff, ndof) small enough for color_exact."""
    out = []
    for name, sub in [("pattern_33_signs20", A.pattern_case(33, "signs20")), ("pattern_2_clamped", A.pattern_case(2, "clamped")),
                      ("duplicate", A.duplicate_case()), ("structure", A.structure_case()), ("no_rows", A.no_rows_case())]:
        out.append((name, C.near_symmetric(sub.groups), sub.loc_dof_eff, sub.ndof))
    return out


def _colour_cases():
    """(name, groups, eff, ndof) of every asm_cases case the coloured operator takes (pattern sizes up to 96)."""
    subs = [(f"pattern_{nd}_{v}", A.pattern_case(nd, v)) for nd in A.PATTERN_SIZES if nd <= 96 for v in A.PATTERN_VARIANTS]
    subs += [("structure", A.structure_case()), ("duplicate", A.duplicate_case()), ("many_groups", A.many_groups_case()),
             ("spd", A.spd_case()), ("order", A.order_case()), ("no_rows", A.no_rows_case())]
    return [(name, C.near_symmetric(s.groups), s.loc_dof_eff, s.ndof) for name, s in subs]


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


@pytest.mark.parametrize("case", range(5))
def test_helper_equals_exact_rational_restatement(case):
    """color_f64 (C, libm fma, no contraction) equals color_exact bit for bit, signed zeros included, in the documented
    order and in both contrasts."""
    from pcg_mpi_solver_b200.coloring import color_groups
    name, groups, eff, ndof = _small_cases()[case]
    colours, _ = color_groups(groups, ndof)
    x = np.random.default_rng(case).standard_normal(len(eff)) * 10.0 ** np.random.default_rng(case).uniform(-3, 3, len(eff))
    for order, scatter in [("documented", "rounded"), ("reversed", "rounded"), ("documented", "contracted")]:
        got = C.color_f64(groups, colours, eff, ndof, x, order, scatter)
        want = C.color_exact(groups, colours, eff, ndof, x, order, scatter)
        assert np.array_equal(_bits(got), _bits(want)), (name, order, scatter)


def test_helper_signed_zeros():
    """x = -0.0 everywhere and a zero Ck: every sum is a zero; the documented sum of zeros from +0.0 stays +0.0."""
    sub = A.pattern_case(31, "signs20")
    groups = C.near_symmetric(sub.groups)
    groups = [dataclasses.replace(groups[0], ck=np.where(np.arange(groups[0].ck.size) % 2 == 0, 0.0, groups[0].ck))]
    from pcg_mpi_solver_b200.coloring import color_groups
    colours, _ = color_groups(groups, sub.ndof)
    x = np.full(sub.n, -0.0)
    got = C.color_f64(groups, colours, sub.loc_dof_eff, sub.ndof, x)
    assert np.array_equal(_bits(got), _bits(C.color_exact(groups, colours, sub.loc_dof_eff, sub.ndof, x)))
    assert np.array_equal(_bits(got), _bits(np.zeros(sub.n)))


def test_helper_tells_the_orders_apart():
    """The helper's sums change under the reversed colour order and under the contracted scatter, on the order pin and
    on cases with many colours per dof."""
    groups, colours, eff, ndof, x, want, rev = C.colour_order_pin()
    assert np.array_equal(C.color_f64(groups, colours, eff, ndof, x), want)
    assert np.array_equal(C.color_f64(groups, colours, eff, ndof, x, order="reversed"), rev)
    assert np.array_equal(C.color_exact(groups, colours, eff, ndof, x), want)
    from pcg_mpi_solver_b200.coloring import color_groups
    for sub in (A.spd_case(), A.duplicate_case()):
        groups = C.near_symmetric(sub.groups)
        colours, nc = color_groups(groups, sub.ndof)
        assert nc > 2
        x = np.random.default_rng(3).standard_normal(sub.n)
        doc = C.color_f64(groups, colours, sub.loc_dof_eff, sub.ndof, x)
        for order, scatter in [("reversed", "rounded"), ("documented", "contracted")]:
            other = C.color_f64(groups, colours, sub.loc_dof_eff, sub.ndof, x, order, scatter)
            assert not np.array_equal(_bits(doc), _bits(other)), (order, scatter)
            assert np.abs(doc - other).max() <= 1e-12 * np.abs(doc).max()


def test_old_colouring_shares_dofs_and_new_colouring_does_not():
    """The first-dof-of-each-triple colouring puts elements that share free dofs in one colour on spd_case (its patterns
    are not node-major); the colouring on every local dof has no conflict on any case, by the library's count and by the
    independent host count."""
    from pcg_mpi_solver_b200.coloring import color_conflicts, color_groups
    sub = A.spd_case()
    old = C.old_colouring(sub.groups, sub.ndof)
    assert C.colour_conflicts(sub.groups, old, sub.loc_dof_eff) > 0
    for name, groups, eff, ndof in _colour_cases():
        colours, nc = color_groups(groups, ndof)
        assert C.colour_conflicts(groups, colours, eff) == 0, name
        em = C._eff_map(eff, ndof)
        assert color_conflicts([em[g.loc_dof] for g in groups], colours, len(eff)) == 0, name
        # the library's count agrees with the host count on the old colouring too
        old = C.old_colouring(groups, ndof)
        assert color_conflicts([em[g.loc_dof] for g in groups], old, len(eff)) == C.colour_conflicts(groups, old, eff), name


def test_node_major_patterns_keep_their_colours():
    """For node-major patterns (the hex and concrete models) the new colouring is the old one, colour for colour."""
    from pcg_mpi_solver_b200.coloring import color_groups
    from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_type_group
    grp, eff, ndof = hex_type_group(HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4), h=0.25))
    new, _ = color_groups([grp], ndof)
    assert np.array_equal(new[0], C.old_colouring([grp], ndof)[0])


@pytest.fixture
def no_library(monkeypatch):
    """Any call into libpcgb200 fails the test."""
    from pcg_mpi_solver_b200 import _lib

    def _refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "load", _refuse)


def test_refusals_happen_before_the_library(no_library):
    """A colouring with a shared dof, a malformed colors_per_group and a non-symmetric Ke raise ValueError in
    EbeMatrixColored before any library call; the library's conflict count matches the host count."""
    from pcg_mpi_solver_b200.coloring import color_conflicts
    from pcg_mpi_solver_b200.ebe import EbeMatrixColored
    sub = A.spd_case()
    groups = C.near_symmetric(sub.groups)
    old = C.old_colouring(groups, sub.ndof)
    with pytest.raises(ValueError, match="two elements of one colour"):
        EbeMatrixColored(groups, sub.loc_dof_eff, sub.ndof, device="cpu", colors_per_group=old)
    # one element moved into the colour of a neighbour that shares a dof with it
    sub = A.duplicate_case()
    groups = C.near_symmetric(sub.groups)
    from pcg_mpi_solver_b200.coloring import color_groups
    colours, _ = color_groups(groups, sub.ndof)
    bad = colours[0].astype(np.int64).copy()
    shared = np.intersect1d(groups[0].loc_dof[:, 0], groups[0].loc_dof[:, 1:])
    e = 1 + int(np.nonzero(np.isin(groups[0].loc_dof[:, 1:], shared).any(axis=0))[0][0])
    bad[e] = bad[0]
    em = C._eff_map(sub.loc_dof_eff, sub.ndof)
    n_bad = color_conflicts([em[groups[0].loc_dof]], [bad], sub.n)
    assert n_bad == C.colour_conflicts(groups, [bad], sub.loc_dof_eff) > 0
    with pytest.raises(ValueError, match="two elements of one colour"):
        EbeMatrixColored(groups, sub.loc_dof_eff, sub.ndof, device="cpu", colors_per_group=[bad])
    for colours_bad in ([bad[:-1]], [bad.astype(np.float64)], [bad - bad.max() - 1], [bad, bad]):
        with pytest.raises(ValueError, match="colors_per_group"):
            EbeMatrixColored(groups, sub.loc_dof_eff, sub.ndof, device="cpu", colors_per_group=colours_bad)
    skew = [dataclasses.replace(groups[0], ke=groups[0].ke + np.triu(np.ones_like(groups[0].ke), 1))]
    with pytest.raises(ValueError, match="symmetric"):
        EbeMatrixColored(skew, sub.loc_dof_eff, sub.ndof, device="cpu")
