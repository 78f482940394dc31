"""Host restatements of the node-block SpMV (csrc/spmv.cuh k_spmv_bsr3 / k_spmv_bsr3_vd and their plan), checked on the CPU
(tests/test_nodeblock_cases_cpu.py) and used by the GPU tests (tests/test_gpu_spmv_nodeblock_order.py).

Both consumers sum a row the same way: a block's partial is fma(a2, x2, fma(a1, x1, a0 * x0)) and the node's partials are
added in block order from +0.0.  A node-block tile is a whole number of nodes, so y does not depend on the plan: one fp64
restatement gives the exact bits of y for every tile, ring, group, consumer count and split launch.

- `rows_f64`     y in that order with a singly rounded fma (a small C helper, pinned against `rows_reference`);
- `rows_reference` the same in Python with an exact rational fma, and the wrong orders a kernel change could introduce;
- `order_pin`    a matrix whose rows give the expected bits only in the documented order;
- `vd_runs`      k_vd_runs per tile: segments, words and nodes in runs; `stream_words` the offsets and cap_words;
- `vd_ring`      the ring choice of the dictionary plan (stages, group, producer warps, shared memory);
- `stream_bytes` pcgb_spmv_stream_bytes of a dictionary plan."""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
import tempfile
from fractions import Fraction

import numpy as np

from tests import spmv_cases as C

EPS = 2.0 ** -53
SEG_CAP = 8            # kVdSegCap
MAX_STAGES = 16        # kBsrMaxStages
VD_STRIDE = 10         # kVdStride
SMEM_CTA = 226 * 1024  # largest dynamic shared memory the plan gives one CTA
SMEM_SM = 227 * 1024   # shared memory per SM


# ------------------------------------------------------------------------------------------------ exact fma
def fma_exact(a, b, c):
    """a * b + c rounded once (to nearest even), with IEEE signs of zero: an exact zero is -0.0 only when a * b and c are
    both zeros of negative sign."""
    r = Fraction(a) * Fraction(b) + Fraction(c)
    if r != 0:
        return float(r)
    if (a == 0 or b == 0) and c == 0:
        pneg = (math.copysign(1.0, a) * math.copysign(1.0, b)) < 0
        return -0.0 if pneg and math.copysign(1.0, c) < 0 else 0.0
    return 0.0


def _row_blocks(indptr, indices, data, r):
    """(values, columns) of row r as (blocks, 3) arrays."""
    a, e = int(indptr[r]), int(indptr[r + 1])
    return np.asarray(data[a:e], dtype=np.float64).reshape(-1, 3), np.asarray(indices[a:e], dtype=np.int64).reshape(-1, 3)


def rows_reference(A, x, rows=None, nest="doc", order="fwd", start=0.0):
    """y[rows] in Python floats with `fma_exact`.  nest: "doc" fma(a2, x2, fma(a1, x1, a0 x0)), "rev" fma(a0, x0, fma(a1,
    x1, a2 x2)), "nofma" (a0 x0 + a1 x1) + a2 x2; order: block order "fwd" or "rev"; start: the accumulator's first value."""
    A = A.tocsr()
    rows = np.arange(A.shape[0]) if rows is None else np.asarray(rows)
    out = np.empty(rows.size)
    for o, r in enumerate(rows):
        v, c = _row_blocks(A.indptr, A.indices, A.data, int(r))
        parts = []
        for (a0, a1, a2), (c0, c1, c2) in zip(v.tolist(), c.tolist()):
            x0, x1, x2 = float(x[c0]), float(x[c1]), float(x[c2])
            if nest == "doc":
                p = fma_exact(a2, x2, fma_exact(a1, x1, a0 * x0))
            elif nest == "rev":
                p = fma_exact(a0, x0, fma_exact(a1, x1, a2 * x2))
            else:
                p = (a0 * x0 + a1 * x1) + a2 * x2
            parts.append(p)
        acc = start
        for p in (parts if order == "fwd" else parts[::-1]):
            acc = acc + p
        out[o] = acc
    return out


_C_SRC = r"""
#include <math.h>
#include <stdint.h>
/* row i of a CSR made of aligned column triples: block partials fma(a2, x2, fma(a1, x1, a0 * x0)) added in order from +0.0 */
void rows_f64(int64_t nr, const int64_t *ip, const int64_t *col, const double *val, const double *x, double *y) {
  for (int64_t i = 0; i < nr; ++i) {
    double acc = 0.0;
    for (int64_t k = ip[i]; k < ip[i + 1]; k += 3) {
      const double p = fma(val[k + 2], x[col[k + 2]], fma(val[k + 1], x[col[k + 1]], val[k] * x[col[k]]));
      acc = acc + p;
    }
    y[i] = acc;
  }
}
/* a[i] * b[i] = p[i] + e[i] exactly */
void two_prod(int64_t n, const double *a, const double *b, double *p, double *e) {
  for (int64_t i = 0; i < n; ++i) { p[i] = a[i] * b[i]; e[i] = fma(a[i], b[i], -p[i]); }
}
"""
_HELPER = None


def _helper():
    """The C helper, compiled once per process into a temporary directory (no contraction, no fast-math)."""
    global _HELPER
    if _HELPER is None:
        d = tempfile.mkdtemp(prefix="nodeblock_rows_")
        src, so = os.path.join(d, "rows.c"), os.path.join(d, "rows.so")
        with open(src, "w") as f:
            f.write(_C_SRC)
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"], check=True)
        lib = ctypes.CDLL(so)
        P = ctypes.c_void_p
        lib.rows_f64.argtypes = [ctypes.c_int64, P, P, P, P, P]
        lib.two_prod.argtypes = [ctypes.c_int64, P, P, P, P]
        _HELPER = lib
    return _HELPER


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def rows_f64_csr(indptr, indices, data, x):
    """y of every row of a (sub-)CSR whose columns index x, in the documented order."""
    ip = np.ascontiguousarray(indptr, dtype=np.int64)
    ip = ip - ip[0]
    col = np.ascontiguousarray(indices, dtype=np.int64)
    val = np.ascontiguousarray(data, dtype=np.float64)
    xx = np.ascontiguousarray(x, dtype=np.float64)
    assert col.size == val.size == ip[-1] and (col.size == 0 or (col.min() >= 0 and col.max() < xx.size))
    y = np.empty(ip.size - 1)
    _helper().rows_f64(y.size, _ptr(ip), _ptr(col), _ptr(val), _ptr(xx), _ptr(y))
    return y


def rows_f64(A, x, rows=None):
    """y[rows] of the node-block CSR A in the documented order (every row when rows is None)."""
    A = A.tocsr()
    if rows is None:
        return rows_f64_csr(A.indptr, A.indices, A.data, x)
    rows = np.asarray(rows, dtype=np.int64)
    a, e = A.indptr[rows].astype(np.int64), A.indptr[rows + 1].astype(np.int64)
    take = np.concatenate([np.arange(s, t) for s, t in zip(a, e)]) if rows.size else np.zeros(0, np.int64)
    ip = np.concatenate([[0], np.cumsum(e - a)])
    return rows_f64_csr(ip, A.indices[take], A.data[take], x)


def exact_dot(x, y):
    """(x . y correctly rounded, sum |x_r y_r|): every product split exactly into p + e, then math.fsum."""
    xx, yy = np.ascontiguousarray(x, dtype=np.float64), np.ascontiguousarray(y, dtype=np.float64)
    p, e = np.empty_like(xx), np.empty_like(xx)
    _helper().two_prod(xx.size, _ptr(xx), _ptr(yy), _ptr(p), _ptr(e))
    return math.fsum(np.concatenate([p, e]).tolist()), float(np.abs(p).sum())


def signed_x(n, seed):
    """x with signed zeros and values over many decades (every 7th entry -0.0, every 11th +0.0, magnitudes 1e-90..1e90)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-90, 91, n)
    x[::7] = -0.0
    x[3::11] = 0.0
    return x


# ------------------------------------------------------------------------------------------------ order pin
ORDER_KINDS = ("order-a", "order-b", "nest", "nofma", "negzero", "empty", "plain")


def order_pin(nn=240):
    """(A, x, kind per node): a chain of nodes coupled to i-1, i, i+1 (interior nodes: three blocks), x = (1, 1, u) on every
    column node, u = 1 + 2^-30.  Node kinds, in turn:
      order-a / order-b  row partials (1, 2^53, -2^53) and (2^53, 1, -2^53): block order gives 0, reversed order 1;
      nest     every block row (2^53, -2^53, 1): fma(a2, x2, fma(a1, x1, a0 x0)) = u, the other nesting 1;
      nofma    blocks rows (-(1 + 2^-29), 0, u), (0, 0, 0), (0, 0, 0): the fma keeps u^2 - (1 + 2^-29) = 2^-60;
      negzero  every value -0.0: partials -0.0, whose sum from +0.0 is +0.0;
      empty    no block at all (y = +0.0);
      plain    random values."""
    rng = np.random.default_rng(21)
    kinds = [ORDER_KINDS[i % len(ORDER_KINDS)] for i in range(nn)]
    nbrs = []
    for i in range(nn):
        cols = np.array([j for j in (i - 1, i, i + 1) if 0 <= j < nn])
        if kinds[i] in ("order-a", "order-b", "nest") and cols.size < 3:
            kinds[i] = "plain"
        nbrs.append(cols if kinds[i] != "empty" else np.zeros(0, np.int64))
    A = C.node_block(nbrs, nn, rng)
    ip = A.indptr
    big, u = 2.0 ** 53, 1.0 + 2.0 ** -30
    for i, k in enumerate(kinds):
        if k in ("plain", "empty"):
            continue
        for r in range(3 * i, 3 * i + 3):
            v = A.data[ip[r]:ip[r + 1]].reshape(-1, 3)
            v[:] = 0.0
            if k == "order-a":
                v[:, 0] = (1.0, big, -big)
            elif k == "order-b":
                v[:, 0] = (big, 1.0, -big)
            elif k == "nest":
                v[:] = (big, -big, 1.0)
            elif k == "nofma":
                v[0] = (-(1.0 + 2.0 ** -29), 0.0, u)
            else:
                v[:] = -0.0
    x = np.tile([1.0, 1.0, u], nn)
    return A, x, np.array(kinds)


# ------------------------------------------------------------------------------------------------ run stream (k_vd_runs)
def _block_positions(A):
    """(blocks, 9) positions in A.data of the 9 values of every 3x3 block, in block order (node, then column)."""
    ip = A.indptr.astype(np.int64)
    a0 = ip[0:-1:3]
    L = ip[1::3] - a0
    nb = L // 3
    node = np.repeat(np.arange(nb.size), nb)
    t = np.arange(node.size) - np.repeat(np.cumsum(nb) - nb, nb)
    base = a0[node] + 3 * t
    r, c = np.repeat(np.arange(3), 3), np.tile(np.arange(3), 3)
    return base[:, None] + r[None, :] * L[node][:, None] + c[None, :]


def node_joins(A):
    """join[i]: node i has node i - 1's block count, and each of its blocks has the bits of the predecessor's block at the
    same place and a column 3 further (the staged x position + 3 of k_vd_runs: both lie in one x window)."""
    A = A.tocsr()
    ip = A.indptr.astype(np.int64)
    nn = (ip.size - 1) // 3
    nb = (ip[1::3] - ip[0:-1:3]) // 3
    pos = _block_positions(A)
    bits = A.data.view(np.int64)[pos]
    bcol = A.indices.astype(np.int64)[pos[:, 0]] if pos.size else np.zeros(0, np.int64)
    node = np.repeat(np.arange(nn), nb)
    same = np.zeros(nn, dtype=bool)
    same[1:] = nb[1:] == nb[:-1]
    g = np.arange(node.size)
    okb = np.zeros(node.size, dtype=bool)
    m = same[node]
    prev = g[m] - nb[node[m]]
    okb[m] = (bcol[g[m]] == bcol[prev] + 3) & (bits[g[m]] == bits[prev]).all(axis=1)
    bad = np.bincount(node[~okb], minlength=nn) if node.size else np.zeros(nn, np.int64)
    return same & (bad == 0), nb


def vd_runs(A, tile_starts, cap=SEG_CAP):
    """k_vd_runs restated on tiles [tile_starts[b], tile_starts[b + 1]) (node indices).  Returns (segs, words, covered):
    segs[b] = [(first node of the tile's segment, is a run)], words[b] = the tile's u32 words (header 1 + 2 per segment +
    the head's blocks of a run / every block of an explicit segment), covered[b] = the tile's nodes in run segments.  A
    tile of more than `cap` segments is one explicit segment with no run."""
    join, nb = node_joins(A)
    starts = np.asarray(tile_starts, dtype=np.int64)
    segs, words, covered = [], np.zeros(starts.size - 1, np.int64), np.zeros(starts.size - 1, np.int64)
    for b, (s, e) in enumerate(zip(starts[:-1], starts[1:])):
        sg, cov = [], 0
        for i in range(s, e):
            if i > s and join[i]:
                cov += 1
                continue
            head = bool(i + 1 < e and join[i + 1])
            if not head and sg and not sg[-1][1]:
                continue
            sg.append((int(i - s), head))
            cov += head
        if len(sg) > cap:
            sg, cov = ([(0, False)] if e > s else []), 0
        nw = 1 + 2 * len(sg)
        for k, (f, run) in enumerate(sg):
            last = sg[k + 1][0] if k + 1 < len(sg) else e - s
            nw += int(nb[s + f]) if run else int(nb[s + f:s + last].sum())
        segs.append(sg)
        words[b], covered[b] = nw, cov
    return segs, words, covered


def stream_words(words):
    """(nvwords, cap_words) of build_vd_runs: the total, and the largest tile slice as the producer's 16-byte aligned
    window (at least 4 words)."""
    w = np.asarray(words, dtype=np.int64)
    end = np.cumsum(w)
    start = end - w
    cap = int(max(4, ((((end + 3) & ~3) - (start & ~3)).max(initial=0))))
    return int(end[-1]) if end.size else 0, cap


def expected_run_nodes(A, tile_items, cap=SEG_CAP):
    """Nodes in run segments of the plan's tiles (k_partition restated by spmv_cases.tile_row_starts)."""
    starts = C.tile_row_starts(A.tocsr().indptr, tile_items, unit=3) // 3
    return int(vd_runs(A, starts, cap)[2].sum())


# ------------------------------------------------------------------------------------------------ ring (build_plan_t)
def producers(stages):
    """Producer warps of a ring: stages % producers == 0, at most 4."""
    return stages if stages < 4 else 4 if stages % 4 == 0 else 2 if stages % 2 == 0 else 1


def vd_ring(cap_x, cap_nodes, cap_words, vd, cw, ctas_per_sm, env_stages=0):
    """The ring of the dictionary plan, or None when no ring fits (the plan then drops the dictionary).  A stage holds sx,
    the node offsets, the tile's words and the meta block; behind the ring sit the y buffers of two groups of G tiles and
    the dictionary.  Default: G = CW down to 1, even rings from min(2 G + 2, 16) down to G + 2, the first that fits the
    plan's CTAs per SM.  env_stages > 0 (PCGB_SPMV_STAGES) forces min(env, 16) stages and G = min(CW, stages)."""
    vstage = (cap_x * 8 + (cap_nodes + 2) * 8 + cap_words * 4 + 32 + 127) & ~127

    def smem(g, s):
        return s * vstage + 2 * g * 3 * cap_nodes * 8 + VD_STRIDE * 8 * vd

    def fits(m):
        return m <= SMEM_CTA and SMEM_SM // (m + 2048) >= ctas_per_sm

    choice = None
    if env_stages > 0:
        s = min(env_stages, MAX_STAGES)
        g = min(cw, s)
        choice = (s, g) if fits(smem(g, s)) else None
    else:
        for g in range(cw, 0, -1):
            for s in range(min((2 * g + 3) & ~1, MAX_STAGES), g + 1, -2):
                if fits(smem(g, s)):
                    choice = (s, g)
                    break
            if choice:
                break
    if choice is None:
        return None
    s, g = choice
    return {"stages": s, "group": g, "producers": producers(s), "stage_bytes": vstage, "smem": smem(g, s)}


# ------------------------------------------------------------------------------------------------ stream bytes
def stream_bytes(info, vd, nvwords, nrows, ncols, rp64):
    """pcgb_spmv_stream_bytes of a persistent dictionary plan: the dictionary once per resident CTA, 4 B per word + 8 B per
    tile of the index stream, row offsets, x, y, the x windows and the tile tables."""
    assert vd > 0 and info["staged"] == 2
    nt = info["ntiles"]
    return (72 * vd * info["resident_ctas"] + 4 * nvwords + 8 * nt + (8 if rp64 else 4) * (nrows + 1) + 8 * ncols + 8 * nrows
            + 8 * info["x_windows"] + 8 * nt + 32 * nt)
