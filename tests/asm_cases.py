"""Seeded pattern-group cases placed on the edges of the device CSR assembly (csrc/assemble.cuh), and a long-double per-row
reference of what it assembles.  numpy only: the cases are checked on the CPU (tests/test_asm_cases_cpu.py) and assembled
on the GPU (tests/test_gpu_assemble_edges.py).

A case is a SubdomainData whose pattern groups put row candidate counts (incident elements x pattern size), distinct
column counts, pattern sizes, key fields (group, element, local index), scan lengths and summation orders where the
kernels branch, overflow or reorder.  The assembled operator is  A = K[Eff,Eff],  K = sum_e P_e^T (Ck_e S_e Ke S_e) P_e.
"""
from __future__ import annotations

import numpy as np

from pcg_mpi_solver_b200.partition import SubdomainData, TypeGroup

MAX_CAND = 2048                 # kAsmMaxCand: candidate columns of one row
PATTERN_SIZES = (1, 2, 31, 32, 33, 64, 65, 127, 128, 129, 254, 255)
PATTERN_VARIANTS = ("plain", "signs20", "signsall", "ck4", "clamped")
BITONIC_TOTALS = (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025)
SCAN_SIZES = (1023, 1024, 1025, 2**20 - 1, 2**20, 2**20 + 1, 3 * 2**20 + 17)
BIG_NE = 2**24 + 3              # element indices >= 2^24 set key bits >= 32
GROUPS_300 = 300                # group indices >= 256 set key bits >= 56
BAND_STRIDE, BAND_ND = 128, 255


def make_sub(groups, ndof, eff) -> SubdomainData:
    eff = np.asarray(eff, dtype=np.int64)
    return SubdomainData(0, 1, np.arange(ndof), np.arange(ndof // 3), eff, groups, [], [], [], np.ones(ndof), np.zeros(ndof),
                         np.zeros(ndof), eff.size, ndof)


def make_group(t, loc, ke, ck, sign=None) -> TypeGroup:
    loc = np.asarray(loc, dtype=np.int64)
    sign = np.zeros(loc.shape, dtype=bool) if sign is None else np.asarray(sign, dtype=bool)
    return TypeGroup(t, loc, sign, np.asarray(ck, dtype=np.float64), np.asarray(ke, dtype=np.float64), np.arange(loc.shape[1]))


def distinct_columns(rng, pool, nd, ne):
    """(nd, ne) dofs drawn from `pool`, distinct within every element."""
    pool = np.asarray(pool, dtype=np.int64)
    if ne == 0:
        return np.zeros((nd, 0), dtype=np.int64)
    return pool[rng.random((ne, pool.size)).argsort(axis=1)[:, :nd].T]


# ----------------------------------------------------------------------------------------- pattern sizes
def pattern_case(nd, variant, seed=0):
    """One group of pattern size nd; every dof is shared by several elements, at most MAX_CAND candidates per row."""
    rng = np.random.default_rng(1000 * nd + PATTERN_VARIANTS.index(variant) + seed)
    ne = min(24, MAX_CAND // nd)
    ndof = nd + max(4, nd // 2)
    loc = distinct_columns(rng, np.arange(ndof), nd, ne)
    ck = rng.permutation(np.logspace(-2, 2, ne)) if variant == "ck4" else rng.random(ne) + 0.5
    sign = {"signs20": rng.random((nd, ne)) < 0.2, "signsall": np.ones((nd, ne), bool)}.get(variant)
    eff = np.arange(ndof)
    if variant == "clamped":
        loc = np.concatenate([loc, np.arange(ndof, ndof + nd)[:, None]], axis=1)      # one element on clamped dofs only
        ck = np.append(ck, 1.0)
        ndof += nd
        eff = np.arange(ndof - nd)
        drop = rng.choice(eff.size, max(1, eff.size // 10), replace=False)
        eff = np.delete(eff, drop)
    return make_sub([make_group(0, loc, rng.standard_normal((nd, nd)), ck, sign)], ndof, eff)


# ----------------------------------------------------------------------------------------- candidate count limit
def candidate_case(total, seed=0):
    """Dof 0 lies in elements whose pattern sizes add up to `total` (2047, 2048 or 2049)."""
    rng = np.random.default_rng(seed + total)
    pool = np.arange(1, 401)
    sizes = {2048: [128] * 16, 2047: [128] * 15 + [127], 2049: [128] * 16 + [1]}[total]
    groups = []
    for t, nd in enumerate(sorted(set(sizes), reverse=True)):
        ne = sizes.count(nd)
        loc = distinct_columns(rng, pool, nd, ne)
        loc[rng.integers(0, nd, ne), np.arange(ne)] = 0
        groups.append(make_group(t, loc, rng.standard_normal((nd, nd)), rng.random(ne) + 0.5, rng.random((nd, ne)) < 0.2))
    return make_sub(groups, 401, np.arange(401))


# ----------------------------------------------------------------------------------------- bitonic / compaction sizes
def _star_sizes(total, k):
    return [total // k + (1 if i < total % k else 0) for i in range(k)]


def bitonic_stars():
    """(total candidates, distinct columns) of the star rows: every BITONIC_TOTALS value with all other columns
    distinct, and for every multiple 32m <= 1024 the distinct counts 32m - 1, 32m, 32m + 1 (8 candidates more)."""
    stars = []
    for T in BITONIC_TOTALS:
        k = -(-T // 128)
        stars.append((T, T - k + 1))
    for m in range(1, 33):
        for D in (32 * m - 1, 32 * m, 32 * m + 1):
            T = D + 8
            stars.append((T, D))
    return stars


def bitonic_case(seed=0):
    """One star per (T, D) of bitonic_stars(): its centre dof lies in k elements of sizes adding up to T (so the row's
    candidate list pads to the next power of two >= T), whose other dofs cycle through a private pool of D - 1 dofs."""
    rng = np.random.default_rng(seed + 7)
    cols = {}                                   # nd -> list of element columns
    nxt = 0
    centres = []
    for T, D in bitonic_stars():
        k = max(-(-T // 128), 1 if T == D else 2)
        sizes = _star_sizes(T, k)
        assert max(sizes) <= D <= T - k + 1, (T, D, sizes)
        r, pool = nxt, np.arange(nxt + 1, nxt + D)
        nxt += D
        centres.append(r)
        off = 0
        for s in sizes:
            other = pool[(off + np.arange(s - 1)) % max(pool.size, 1)] if s > 1 else np.zeros(0, np.int64)
            off += s - 1
            col = np.insert(other, rng.integers(0, s), r)
            cols.setdefault(s, []).append(col)
    groups = []
    for t, nd in enumerate(sorted(cols)):
        loc = np.stack(cols[nd], axis=1)
        ne = loc.shape[1]
        groups.append(make_group(t, loc, rng.standard_normal((nd, nd)), rng.random(ne) + 0.5, rng.random((nd, ne)) < 0.2))
    sub = make_sub(groups, nxt, np.arange(nxt))
    sub.extra["centres"] = np.array(centres)
    return sub


# ----------------------------------------------------------------------------------------- structural edges
def structure_case(seed=0):
    """Empty rows (start, middle, end), rows whose elements touch only clamped dofs besides the diagonal, groups with
    ne = 0 between others, and a hub dof shared by 200 elements of size 10 (2000 candidates, a 200-entry insertion sort)."""
    rng = np.random.default_rng(seed + 11)
    ndof = 520
    empty = np.array([0, 260, ndof - 1])                 # free, untouched
    clamped = np.arange(500, 519)                         # not free
    lonely = np.array([300, 301])                         # free; their elements' other dofs are all clamped
    hub = 150
    pool = np.setdiff1d(np.arange(ndof), np.concatenate([empty, clamped, lonely, [hub]]))
    groups = []
    g0 = distinct_columns(rng, np.concatenate([pool, clamped[:5]]), 5, 30)
    g1 = distinct_columns(rng, pool, 3, 40)
    g_lonely = np.concatenate([distinct_columns(rng, clamped, 5, 4), np.repeat(lonely, 2)[None, :]], axis=0)   # (6, 4)
    g_hub = distinct_columns(rng, pool, 9, 200)
    g_hub = np.concatenate([g_hub[:4], np.full((1, 200), hub), g_hub[4:]], axis=0)                              # (10, 200)
    empty_nd = iter((7, 2, 9))
    for loc in (g0, None, g1, g_lonely, None, g_hub, None):
        nd = next(empty_nd) if loc is None else loc.shape[0]
        loc = np.zeros((nd, 0), np.int64) if loc is None else loc
        ne = loc.shape[1]
        groups.append(make_group(len(groups), loc, rng.standard_normal((nd, nd)), rng.random(ne) + 0.5, rng.random((nd, ne)) < 0.2))
    eff = np.setdiff1d(np.arange(ndof), clamped)
    sub = make_sub(groups, ndof, eff)
    sub.extra.update(empty=empty, lonely=lonely, hub=hub)
    return sub


def no_rows_case(seed=0):
    """n = 0: every dof clamped (the elements are still there)."""
    rng = np.random.default_rng(seed + 13)
    loc = distinct_columns(rng, np.arange(40), 6, 10)
    return make_sub([make_group(0, loc, rng.standard_normal((6, 6)), rng.random(10) + 0.5)], 40, np.zeros(0, np.int64))


# ----------------------------------------------------------------------------------------- key fields
def many_groups_case(seed=0):
    """GROUPS_300 groups of one shape (nd 4, ne 3) on 120 dofs: every row mixes groups below and above 256."""
    rng = np.random.default_rng(seed + 17)
    groups = [make_group(t, distinct_columns(rng, np.arange(120), 4, 3), rng.standard_normal((4, 4)), rng.random(3) + 0.5,
                         rng.random((4, 3)) < 0.2) for t in range(GROUPS_300)]
    return make_sub(groups, 120, np.arange(120))


def many_elements_case(seed=0):
    """One nd = 1 group of BIG_NE elements spread over 2^22 dofs (about 4 per dof)."""
    rng = np.random.default_rng(seed + 19)
    ndof = 2**22
    loc = rng.integers(0, ndof, BIG_NE)[None, :]
    return make_sub([make_group(0, loc, [[1.5]], rng.random(BIG_NE) + 0.5)], ndof, np.arange(ndof))


def wide_pattern_case(seed=0):
    """nd = 255 (local index 255 fills the 8-bit key field) with signs, 8 elements on 300 dofs."""
    rng = np.random.default_rng(seed + 23)
    loc = distinct_columns(rng, np.arange(300), 255, 8)
    return make_sub([make_group(0, loc, rng.standard_normal((255, 255)), rng.random(8) + 0.5, rng.random((255, 8)) < 0.2)],
                    300, np.arange(300))


# ----------------------------------------------------------------------------------------- scan lengths
def scan_case(n, seed=0):
    """n free dofs under nd 3 / nd 4 elements placed at random, about one element per dof: row lengths vary from 0 up."""
    rng = np.random.default_rng(seed + n)
    groups = []
    for t, nd in enumerate((3, 4)):
        ne = n // 7
        start = rng.integers(0, n - 8, ne)
        loc = start[None, :] + np.argsort(rng.random((ne, 8)), axis=1)[:, :nd].T      # nd distinct dofs in a window of 8
        loc[:, 0] = n - nd + np.arange(nd)                                              # the last rows are never empty
        groups.append(make_group(t, loc, rng.standard_normal((nd, nd)), rng.random(ne) + 0.5, rng.random((nd, ne)) < 0.2))
    return make_sub(groups, n, np.arange(n))


# ----------------------------------------------------------------------------------------- summation order
ORDER_ND, ORDER_NE = 8, 2048


def order_case(seed=0):
    """Rows whose diagonal sums 2^53, 1, -2^53 (exact products: Ke small integers, Ck powers of two).  Row r lies at local
    index 7 of element a, 4 of element b and 0 of element c, a < b < c: the documented order (group, element, local index)
    adds a, b, c -> 0, while k_asm_fill (thread i * ne + e) reaches them as c, b, a -> 1."""
    rng = np.random.default_rng(seed + 29)
    nd, ne = ORDER_ND, ORDER_NE
    rows = np.array([0, 1, 2])
    pool = np.arange(3, 603)
    loc = distinct_columns(rng, pool, nd, ne)
    ck = 2.0 ** rng.integers(-2, 3, ne)
    ke = rng.integers(-3, 4, (nd, nd)).astype(float)
    ke = ke + ke.T
    ke[7, 7], ke[4, 4], ke[0, 0] = 1.0, 1.0, -1.0
    for q, r in enumerate(rows):
        a, b, c = 100 * q + 5, 100 * q + 40, 100 * q + 90
        loc[7, a], loc[4, b], loc[0, c] = r, r, r
        ck[a], ck[b], ck[c] = 2.0**53, 1.0, 2.0**53
    sign = rng.random((nd, ne)) < 0.2
    sub = make_sub([make_group(0, loc, ke, ck, sign)], 603, np.arange(603))
    sub.extra["rows"] = rows
    return sub


# ----------------------------------------------------------------------------------------- repeated dofs in one element
DUP_ND = 40


def duplicate_case(seed=0):
    """nd = 40 elements listing a free dof twice: at local indices 3 and 10 (one 32-lane pass), at 5 and 38 (passes j and
    j + 32 on different lanes), and three times at 1, 2 and 33; the last elements have no repeats."""
    rng = np.random.default_rng(seed + 31)
    nd, ne = DUP_ND, 60
    loc = distinct_columns(rng, np.arange(200), nd, ne)
    loc[10, 0:20] = loc[3, 0:20]
    loc[38, 20:40] = loc[5, 20:40]
    loc[2, 40:50] = loc[1, 40:50]
    loc[33, 40:50] = loc[1, 40:50]
    eff = np.setdiff1d(np.arange(200), rng.choice(200, 15, replace=False))
    return make_sub([make_group(0, loc, rng.standard_normal((nd, nd)), rng.random(ne) + 0.5, rng.random((nd, ne)) < 0.2)], 200, eff)


# ----------------------------------------------------------------------------------------- SPD system for the solver
def spd_case(seed=0):
    """Sum of PSD element matrices (sizes 24 and 40, signs) plus an nd = 1 group on every dof with positive Ck: SPD on the
    free dofs."""
    rng = np.random.default_rng(seed + 37)
    ndof = 900
    groups = []
    for t, (nd, ne) in enumerate(((24, 120), (40, 30))):
        B = rng.standard_normal((nd, nd))
        groups.append(make_group(t, distinct_columns(rng, np.arange(ndof), nd, ne), B @ B.T / nd, rng.random(ne) + 0.5,
                                 rng.random((nd, ne)) < 0.2))
    groups.append(make_group(2, np.arange(ndof)[None, :], [[1.0]], 0.05 + 0.1 * rng.random(ndof)))
    eff = np.setdiff1d(np.arange(ndof), rng.choice(ndof, 60, replace=False))
    return make_sub(groups, ndof, eff)


# ----------------------------------------------------------------------------------------- int64 row offsets
def band_case(ne, seed=0):
    """One nd = 255 group, element e on dofs [128 e, 128 e + 255): every row has 255 or 383 columns."""
    rng = np.random.default_rng(seed + 41)
    ndof = BAND_STRIDE * (ne - 1) + BAND_ND
    loc = BAND_STRIDE * np.arange(ne)[None, :] + np.arange(BAND_ND)[:, None]
    ke = rng.standard_normal((BAND_ND, BAND_ND))
    return make_sub([make_group(0, loc, ke, rng.random(ne) + 0.5, rng.random((BAND_ND, ne)) < 0.2)], ndof, np.arange(ndof))


def band_row_lengths(ne):
    """Row lengths of band_case(ne), analytically: dof d lies in elements ceil((d - 254) / 128) .. floor(d / 128)."""
    d = np.arange(BAND_STRIDE * (ne - 1) + BAND_ND, dtype=np.int64)
    e_lo = np.maximum(0, -(-(d - (BAND_ND - 1)) // BAND_STRIDE))
    e_hi = np.minimum(ne - 1, d // BAND_STRIDE)
    return BAND_STRIDE * (e_hi - e_lo) + BAND_ND


# band_case(INT64_NE) has more than 2^31 non-zeros
INT64_NE = 44_000


# ----------------------------------------------------------------------------------------- what the cases reach
def candidates(sub):
    """Per free row: sum of the pattern sizes of its incident (element, local index) pairs - the kernel's candidate count."""
    pos = np.full(sub.ndof, -1, np.int64)
    pos[sub.loc_dof_eff] = np.arange(sub.n)
    c = np.zeros(sub.ndof, np.int64)
    for g in sub.groups:
        c += np.bincount(g.loc_dof.ravel(), minlength=sub.ndof) * g.loc_dof.shape[0]
    return c[sub.loc_dof_eff]


# ----------------------------------------------------------------------------------------- reference
def _terms(sub, rows):
    """Every term (s_i s_j) Ke[i][j] Ck_e of the rows `rows` (sorted, unique free indices) with its slot in `rows`, its free
    column and its documented-order key (group, element, local index i, local index j) and fill-order key (group,
    i * ne + e, j)."""
    n = sub.n
    pos = np.full(sub.ndof, -1, np.int64)
    pos[sub.loc_dof_eff] = np.arange(n)
    slot = np.full(n + 1, -1, np.int64)
    slot[rows] = np.arange(rows.size)
    out = []
    for gi, g in enumerate(sub.groups):
        nd, ne = g.loc_dof.shape
        if ne == 0:
            continue
        p = pos[g.loc_dof]
        w = slot[p]                                            # p = -1 -> slot[n] = -1
        ii, ee = np.nonzero(w >= 0)
        if ii.size == 0:
            continue
        cols = p[:, ee].T                                      # (m, nd)
        s = np.where(g.sign, -1, 1).astype(np.int8)
        sg = s[ii, ee][:, None] * s[:, ee].T
        t = (sg * g.ke[ii, :]).astype(np.longdouble) * g.ck[ee].astype(np.longdouble)[:, None]
        keep = cols >= 0
        jj = np.broadcast_to(np.arange(nd), cols.shape)
        out.append(dict(slot=np.broadcast_to(w[ii, ee][:, None], cols.shape)[keep], col=cols[keep], t=t[keep], g=np.full(keep.sum(), gi),
                        e=np.broadcast_to(ee[:, None], cols.shape)[keep], i=np.broadcast_to(ii[:, None], cols.shape)[keep], j=jj[keep],
                        ne=np.full(keep.sum(), ne)))
    if not out:
        z = np.zeros(0, np.int64)
        return dict(slot=z, col=z, t=np.zeros(0, np.longdouble), g=z, e=z, i=z, j=z, ne=z)
    return {k: np.concatenate([o[k] for o in out]) for k in out[0]}


def ref_rows(sub, rows=None):
    """Long-double restatement of  K[Eff,Eff] = sum_e P_e^T (Ck_e S_e Ke S_e) P_e  on the free rows `rows` (all by default).
    Returns (rows, indptr, col, val, abs_sum, count): per row the distinct free columns ascending, and per entry the value,
    sum |terms| and number of terms, for the bound |val - ref| <= (count + 2) 2^-53 abs_sum."""
    rows = np.arange(sub.n, dtype=np.int64) if rows is None else np.unique(np.asarray(rows, dtype=np.int64))
    T = _terms(sub, rows)
    key = T["slot"] * max(sub.n, 1) + T["col"]
    o = np.argsort(key, kind="stable")
    key, t = key[o], T["t"][o]
    if key.size == 0:
        z = np.zeros(0, np.int64)
        return rows, np.zeros(rows.size + 1, np.int64), z, np.zeros(0, np.longdouble), np.zeros(0, np.longdouble), z
    first = np.concatenate([[True], key[1:] != key[:-1]])
    starts = np.nonzero(first)[0]
    val = np.add.reduceat(t, starts)
    asum = np.add.reduceat(np.abs(t), starts)
    cnt = np.diff(np.append(starts, key.size))
    uk = key[starts]
    slot, col = uk // max(sub.n, 1), uk % max(sub.n, 1)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(slot, minlength=rows.size))])
    return rows, indptr, col, val, asum, cnt


def ordered_sums(sub, order):
    """fp64 sums per (row, col) of all rows, adding the terms one by one in `order`: "documented" (group, element, local
    index i, then j - the order csrc/assemble.cuh states), "fill" (group, k_asm_fill's thread index i * ne + e, j) or
    "reversed" (documented, backwards).  Returns {(row, col): float}.  For small cases."""
    T = _terms(sub, np.arange(sub.n, dtype=np.int64))
    if order == "fill":
        o = np.lexsort((T["j"], T["i"] * T["ne"] + T["e"], T["g"]))
    else:
        o = np.lexsort((T["j"], T["i"], T["e"], T["g"]))
        if order == "reversed":
            o = o[::-1]
    sums = {}
    for s, c, t in zip(T["slot"][o].tolist(), T["col"][o].tolist(), T["t"][o].astype(np.float64).tolist()):
        sums[(s, c)] = sums.get((s, c), 0.0) + t
    return sums
