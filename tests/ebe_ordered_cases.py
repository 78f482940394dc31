"""Cases and host restatements for the ordered matrix-free operator (csrc/ebe_ordered.cuh, EbeMatrixOrdered).

`ref_apply` restates the operator in long double with the rounding scale of every entry; `ordered_f64` restates it in
fp64 with the documented order of both phases (and, for contrast, the per-element order); `order_pin` is a case whose
phase-1 products are exact and whose per-dof sums cancel differently in every order but the documented one."""
from fractions import Fraction

import numpy as np

from pcg_mpi_solver_b200.partition import TypeGroup

EPS = 2.0 ** -53


def _eff_map(eff, ndof):
    n = len(eff)
    m = np.full(ndof, -1, dtype=np.int64)
    m[np.asarray(eff, dtype=np.int64)] = np.arange(n)
    return m


def ref_apply(groups, eff, ndof, x):
    """(y, abs_sum, count) per free dof in long double: y = sum over the dof's slots of s_a sum_b Ke[a][b] Ck_e s_b x_b,
    abs_sum = the same sum of |terms|, count = number of product terms plus slots.  A computed y is right when
    |y - ref| <= (count + 2) 2^-53 abs_sum."""
    n = len(eff)
    em = _eff_map(eff, ndof)
    xe = np.zeros(n + 1, dtype=np.longdouble)
    xe[:n] = x
    y = np.zeros(n + 1, dtype=np.longdouble)
    b = np.zeros(n + 1, dtype=np.longdouble)
    k = np.zeros(n + 1, dtype=np.int64)
    for g in groups:
        idx = em[g.loc_dof]                                # (nd, ne), -1 clamped
        nd, ne = idx.shape
        if ne == 0:
            continue
        ix = np.where(idx >= 0, idx, n)                    # clamped: gather 0, scatter into a dropped slot
        ke = np.asarray(g.ke, dtype=np.longdouble)
        ck = np.asarray(g.ck, dtype=np.longdouble)
        s = np.where(g.sign, -1.0, 1.0).astype(np.longdouble)
        u = ck[None, :] * (s * xe[ix])
        np.add.at(y, ix, s * (ke @ u))
        np.add.at(b, ix, np.abs(ke) @ np.abs(u))
        np.add.at(k, ix, nd + 1)
    return y[:n], b[:n], k[:n]


def assert_entrywise(y, groups, eff, ndof, x):
    ref, b, k = ref_apply(groups, eff, ndof, x)
    assert not np.isnan(y).any(), f"{int(np.isnan(y).sum())} entries never written"
    err = np.abs(np.asarray(y, dtype=np.longdouble) - ref)
    bad = np.nonzero(err > (k + 2) * EPS * b)[0]
    assert bad.size == 0, f"{bad.size} entries off, first {bad[:5]}: err {err[bad[:5]]} bound {((k + 2) * EPS * b)[bad[:5]]}"


def _fma(a, b, c):
    """a * b + c with one rounding (exact rational arithmetic, rounded once by the float conversion)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def slot_values(groups, eff, ndof, x):
    """Phase 1 in fp64 as documented, for small cases: [(dof, slot position, value, group, element, local index)] for
    every slot of a free local index."""
    em = _eff_map(eff, ndof)
    out, off = [], 0
    for t, g in enumerate(groups):
        idx = em[g.loc_dof]
        nd, ne = idx.shape
        ke = np.asarray(g.ke, dtype=np.float64)
        for e in range(ne):
            u = [float(g.ck[e]) * ((-1.0 if g.sign[b, e] else 1.0) * float(x[idx[b, e]])) if idx[b, e] >= 0 else 0.0
                 for b in range(nd)]
            for a in range(nd):
                if idx[a, e] < 0:
                    continue
                acc = 0.0
                for b in range(nd):
                    acc = _fma(float(ke[a, b]), u[b], acc)
                out.append((int(idx[a, e]), off + a * ne + e, -acc if g.sign[a, e] else acc, t, e, a))
        off += nd * ne
    return out


def ordered_f64(groups, eff, ndof, x, order="documented"):
    """fp64 y with the slots of each dof added from 0.0 in `order`: "documented" (ascending slot position = group, local
    index, element) or "element" (group, element, local index)."""
    key = (lambda v: v[1]) if order == "documented" else (lambda v: (v[3], v[4], v[5]))
    y = np.zeros(len(eff))
    for dof, _, v, *_ in sorted(slot_values(groups, eff, ndof, x), key=key):
        y[dof] = y[dof] + v
    return y


def order_pin():
    """One nd = 2 group, Ke = I, x = 1, integer Ck: every phase-1 product is exact.  Free dof d (d = 0, 1, 2) collects
    the values 2^53, -2^53 and 1 from three slots; the 1 sits at ascending position d + 1.  Adding from 0.0, the 1 survives
    only when it comes last: the documented order gives y = (0, 0, 1), and any order that puts another slot last gives
    another vector.  The per-element order (group, element, local index) gives (1, 1, 0).  Returns (groups, eff, ndof, x,
    expected)."""
    big = 2.0 ** 53
    # element e: local 0 -> dof l0[e] with Ck c[e], local 1 clamped (dof 3) or the same dof as local 0
    # slot positions: a * ne + e.  Per dof the three slots, ascending, with the wanted values.
    want = {0: (1.0, big, -big), 1: (big, 1.0, -big), 2: (big, -big, 1.0)}
    # dof d uses elements 3d .. 3d+2 and local indices chosen so that the ascending order of (a * ne + e) is the listed one:
    # slots (a=0, e=3d+1), (a=0, e=3d+2), (a=1, e=3d): ascending positions e=3d+1, e=3d+2 (a = 0) then 3d (a = 1).
    ne = 9
    loc = np.full((2, ne), 3, dtype=np.int64)          # dof 3 is clamped
    ck = np.zeros(ne)
    for d in range(3):
        first, second, third = want[d]
        loc[0, 3 * d + 1], ck[3 * d + 1] = d, first
        loc[0, 3 * d + 2], ck[3 * d + 2] = d, second
        loc[1, 3 * d], ck[3 * d] = d, third
    g = TypeGroup(0, loc, np.zeros((2, ne), dtype=bool), ck, np.eye(2), np.arange(ne))
    return [g], np.arange(3), 4, np.ones(3), np.array([0.0, 0.0, 1.0])
