"""Host restatements and cases for the coloured matrix-free operator (csrc/ebe_color.cuh, EbeMatrixColored), checked on the
CPU (tests/test_ebe_color_cases_cpu.py) and used by the GPU tests (tests/test_gpu_ebe_color_edges.py).

The documented result (include/pcgb200.h): every free dof d starts from +0.0; the colours are taken in ascending order,
and for the one element e of that colour that touches d, every local index i with idx[i] = d, in ascending i, does
y_d = y_d + v_{e,i}, with u_j = s_j x_j (0.0 for a clamped dof), acc = fma(Ke[i][j], u_j, acc) over j ascending from 0.0
and v_{e,i} = round(acc * Ck_e), negated when s_i is set.  Inside one colour no two elements share a free dof, so the
order of the elements of a colour does not change a bit.

- `color_f64`        that result in fp64 (a small C helper), or with the colours reversed or the scatter contracted;
- `color_exact`      the same in Python with an exact rational fma, for small cases;
- `colour_conflicts` (colour, free dof) pairs touched by two different elements of one colour, with Python sets;
- `old_colouring`    the colouring on the first dof of every triple only, which is right for node-major patterns only;
- `near_symmetric`   a case's pattern matrices made symmetric to within a few ulps but not bit for bit;
- `colour_order_pin` caller-given colours whose sums give the expected vector only in the documented colour order."""
from __future__ import annotations

import ctypes
import dataclasses
import os
import subprocess
import tempfile

import numpy as np

from pcg_mpi_solver_b200.partition import TypeGroup
from tests.nodeblock_cases import fma_exact

_C_SRC = r"""
#include <math.h>
#include <stdint.h>
/* ne elements of one (pattern group, colour) slice: idx (ne, nd) free indices (-1 = clamped), sign (ne, nd), ck (ne),
   ke (nd, nd) row-major.  contract = 0: v = acc * ck, negated for s_i, then y = y + v (two roundings);
   contract = 1: y = fma(+-acc, ck, y) (one rounding). */
void color_slice(int64_t ne, int nd, const int32_t *idx, const uint8_t *sign, const double *ck, const double *ke,
                 const double *x, double *y, int contract) {
  double u[256];
  for (int64_t e = 0; e < ne; ++e) {
    const int32_t *id = idx + e * nd;
    const uint8_t *s = sign + e * nd;
    for (int j = 0; j < nd; ++j) u[j] = id[j] >= 0 ? (s[j] ? -x[id[j]] : x[id[j]]) : 0.0;
    for (int i = 0; i < nd; ++i) {
      double acc = 0.0;
      for (int j = 0; j < nd; ++j) acc = fma(ke[(int64_t)i * nd + j], u[j], acc);
      if (id[i] < 0) continue;
      if (contract) {
        y[id[i]] = fma(s[i] ? -acc : acc, ck[e], y[id[i]]);
      } else {
        double v = acc * ck[e];
        if (s[i]) v = -v;
        y[id[i]] = y[id[i]] + v;
      }
    }
  }
}
"""
_HELPER = None


def _helper():
    """The C helper, compiled once per process into a temporary directory (no contraction, no fast-math)."""
    global _HELPER
    if _HELPER is None:
        d = tempfile.mkdtemp(prefix="ebe_color_")
        src, so = os.path.join(d, "color.c"), os.path.join(d, "color.so")
        with open(src, "w") as f:
            f.write(_C_SRC)
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"], check=True)
        lib = ctypes.CDLL(so)
        P = ctypes.c_void_p
        lib.color_slice.argtypes = [ctypes.c_int64, ctypes.c_int, P, P, P, P, P, P, ctypes.c_int]
        _HELPER = lib
    return _HELPER


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _eff_map(eff, ndof):
    m = np.full(ndof, -1, dtype=np.int64)
    m[np.asarray(eff, dtype=np.int64)] = np.arange(len(eff))
    return m


def _slices(groups, colours, eff, ndof, order):
    """(colour, group index, element indices) of every non-empty slice, colours in `order` ("documented" ascending or
    "reversed"), groups ascending inside a colour."""
    ncol = max([int(np.max(c)) + 1 for c in colours if len(c)], default=0)
    out = []
    for c in (range(ncol) if order == "documented" else range(ncol - 1, -1, -1)):
        for t, col in enumerate(colours):
            sel = np.nonzero(np.asarray(col) == c)[0]
            if sel.size:
                out.append((c, t, sel))
    return out


def color_f64(groups, colours, eff, ndof, x, order="documented", scatter="rounded"):
    """y in fp64 as documented; order="reversed" takes the colours backwards, scatter="contracted" adds every product with
    one rounding, y = fma(+-acc, Ck, y)."""
    lib = _helper()
    em = _eff_map(eff, ndof)
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.zeros(len(eff))
    idx = [np.ascontiguousarray(em[g.loc_dof].T, dtype=np.int32) for g in groups]
    for c, t, sel in _slices(groups, colours, eff, ndof, order):
        g = groups[t]
        nd = g.loc_dof.shape[0]
        ii = np.ascontiguousarray(idx[t][sel])
        ss = np.ascontiguousarray(np.asarray(g.sign)[:, sel].T, dtype=np.uint8)
        ck = np.ascontiguousarray(np.asarray(g.ck, dtype=np.float64)[sel])
        ke = np.ascontiguousarray(g.ke, dtype=np.float64)
        lib.color_slice(sel.size, nd, _ptr(ii), _ptr(ss), _ptr(ck), _ptr(ke), _ptr(x), _ptr(y), int(scatter == "contracted"))
    return y


def color_exact(groups, colours, eff, ndof, x, order="documented", scatter="rounded"):
    """color_f64 in Python floats with `fma_exact` for every operation: a * b = fma(a, b, -0.0), a + b = fma(1, a, b)."""
    em = _eff_map(eff, ndof)
    y = [0.0] * len(eff)
    for c, t, sel in _slices(groups, colours, eff, ndof, order):
        g = groups[t]
        nd = g.loc_dof.shape[0]
        ke = np.asarray(g.ke, dtype=np.float64).tolist()
        for e in sel.tolist():
            id_ = [int(em[g.loc_dof[j, e]]) for j in range(nd)]
            s = [bool(g.sign[j, e]) for j in range(nd)]
            ck = float(g.ck[e])
            u = [(-float(x[id_[j]]) if s[j] else float(x[id_[j]])) if id_[j] >= 0 else 0.0 for j in range(nd)]
            for i in range(nd):
                acc = 0.0
                for j in range(nd):
                    acc = fma_exact(ke[i][j], u[j], acc)
                if id_[i] < 0:
                    continue
                if scatter == "contracted":
                    y[id_[i]] = fma_exact(-acc if s[i] else acc, ck, y[id_[i]])
                else:
                    v = fma_exact(acc, ck, -0.0)
                    y[id_[i]] = fma_exact(1.0, y[id_[i]], -v if s[i] else v)
    return np.array(y, dtype=np.float64)


def colour_conflicts(groups, colours, eff):
    """Number of (colour, free dof) pairs that two different elements of one colour touch (an element's own repeats do
    not count)."""
    pos = {int(d): k for k, d in enumerate(np.asarray(eff).tolist())}
    owner, bad = {}, set()
    for t, (g, col) in enumerate(zip(groups, colours)):
        for e in range(g.loc_dof.shape[1]):
            for d in set(g.loc_dof[:, e].tolist()):
                if d not in pos:
                    continue
                key = (int(col[e]), pos[d])
                if owner.setdefault(key, (t, e)) != (t, e):
                    bad.add(key)
    return len(bad)


def old_colouring(groups, ndof):
    """The colouring on loc_dof[0::3] // 3 (the node of the first dof of every triple) - valid only when local dof j is
    3 node[j // 3] + j % 3."""
    from pcg_mpi_solver_b200.coloring import color_elements
    flat = np.concatenate([(g.loc_dof[0::3, :] // 3).T.ravel() for g in groups])
    counts = np.concatenate([np.full(g.loc_dof.shape[1], (g.loc_dof.shape[0] + 2) // 3, dtype=np.int64) for g in groups])
    colors, _ = color_elements(flat, np.concatenate([[0], np.cumsum(counts)]), ndof // 3 + 1)
    return np.split(colors, np.cumsum([g.loc_dof.shape[1] for g in groups])[:-1])


def near_symmetric(groups, seed=0):
    """The groups with Ke + Ke^T scaled entrywise by 1 + 2^-48 r, r uniform in [-1, 1]: symmetric to well inside
    EbeMatrix's 1e-12 test, but not bit for bit, so a kernel that reads Ke^T instead of Ke changes the result."""
    rng = np.random.default_rng(seed + 101)
    out = []
    for g in groups:
        ke = np.asarray(g.ke, dtype=np.float64)
        ke = (ke + ke.T) * (1.0 + 2.0 ** -48 * rng.uniform(-1.0, 1.0, ke.shape))
        out.append(dataclasses.replace(g, ke=ke))
    return out


def colour_order_pin():
    """Three free dofs, one nd = 1 group with Ke = [[1]], x = 1: element e adds exactly Ck_e to its dof.  Each dof gets
    one element in each of the colours 0, 1, 2, with the values (by colour)
        dof 0: 1, 2^53, -2^53      dof 1: 2^53, 1, -2^53      dof 2: 2^53, -2^53, 1.
    From +0.0, a dof keeps its 1 unless -2^53 is added last, so the documented order gives (0, 0, 1) and exactly the colour
    orders that take colour 2 last give it (the first two additions into +0.0 commute, so no sum can order colours 0 and
    1).  The reversed order gives (1, 1, 1).  Returns (groups, colours, eff, ndof, x, expected, reversed)."""
    big = 2.0 ** 53
    vals = {0: (1.0, big, -big), 1: (big, 1.0, -big), 2: (big, -big, 1.0)}
    loc, ck, col = [], [], []
    for c in (2, 0, 1):                                   # element order inside the group does not follow the colours
        for d in range(3):
            loc.append(d)
            ck.append(vals[d][c])
            col.append(c)
    ne = len(loc)
    g = TypeGroup(0, np.array([loc], dtype=np.int64), np.zeros((1, ne), dtype=bool), np.array(ck), np.ones((1, 1)), np.arange(ne))
    return [g], [np.array(col, dtype=np.int64)], np.arange(3), 3, np.ones(3), np.array([0.0, 0.0, 1.0]), np.array([1.0, 1.0, 1.0])
