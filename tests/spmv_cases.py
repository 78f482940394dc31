"""Seeded CSR test matrices placed on the branch points of the SpMV kernels (csrc/spmv.cuh), and a long-double
reference product.  numpy / scipy only: the generators are checked on the CPU (tests/test_spmv_cases_cpu.py) and
used by the GPU tests (tests/test_gpu_spmv_edges.py).

Node-block ("BSR-3") matrices are a node graph expanded to 3x3 blocks: rows 3n, 3n+1, 3n+2 share one column
pattern made of aligned column triples 3j, 3j+1, 3j+2, which is what the plan checks before it picks k_spmv_bsr3.
Row-group matrices put row lengths, empty rows, long rows and x windows where the row-group kernels branch.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

# node-block plan limit (spmv.cuh, build_plan_t): the kernel needs tile_items >= 2 * 3 * (max_row + 1) with the default tile
# 6100 - 3 * (max_row + 1) (in-place row partials) or 4608 - 3 * (max_row + 1) (PCGB_BSR_INPLACE=0), so the longest row
# may have at most 676 (511) non-zeros, i.e. a node at most 225 (170) blocks
BSR_MAX_ROW = {1: 676, 0: 511}


# ----------------------------------------------------------------------------------------- reference
def ref_spmv(A, x):
    """y = A x summed in long double, and the entrywise scale (|A| |x|)_i of the fp64 rounding bound."""
    A = sp.csr_matrix(A)
    xl = np.asarray(x, dtype=np.longdouble)
    prod = np.append(A.data.astype(np.longdouble) * xl[A.indices], np.longdouble(0))
    starts = np.minimum(A.indptr[:-1], A.nnz)
    y = np.add.reduceat(prod, starts) if A.shape[0] else np.zeros(0, dtype=np.longdouble)
    y[np.diff(A.indptr) == 0] = 0
    scale = abs(A) @ np.abs(np.asarray(x, dtype=np.float64))
    return y, scale


def tile_row_starts(indptr, tile_items, unit=1):
    """First row of every tile (and the end) as the plan's merge-path partition computes it (k_partition with row snap;
    unit = 3 for node-block plans, whose tiles start at a node)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    n, nnz = indptr.size - 1, int(indptr[-1])
    total = n + nnz
    nt = max(1, -(-total // tile_items))
    d = np.minimum(np.arange(nt + 1, dtype=np.int64) * tile_items, total)
    d[-1] = total
    i = np.searchsorted(indptr[1:] + np.arange(1, n + 1), d, side="right")
    i = np.clip(i, np.maximum(0, d - nnz), np.minimum(d, n))
    return np.where(i < n, i - i % unit, i)


# ----------------------------------------------------------------------------------------- node-block matrices
def node_block(nbrs, ncol_nodes, rng, spd=False):
    """Expand node neighbour lists (one sorted array of column nodes per row node) to 3x3 blocks with random values.
    spd: nbrs must be symmetric and contain the diagonal; off-diagonal blocks get B_ji = B_ij^T and every diagonal
    block is made strictly dominant (5 % above the row's off-diagonal absolute sum), so the matrix is SPD."""
    nn = len(nbrs)
    cnt = np.array([len(v) for v in nbrs], dtype=np.int64)
    bi = np.repeat(np.arange(nn), cnt)
    bj = np.concatenate([np.asarray(v, dtype=np.int64) for v in nbrs]) if nn else np.zeros(0, np.int64)
    blocks = rng.standard_normal((bi.size, 3, 3))
    if spd:
        key = {(int(i), int(j)): k for k, (i, j) in enumerate(zip(bi, bj))}
        for k, (i, j) in enumerate(zip(bi, bj)):
            if i > j:
                blocks[k] = blocks[key[(int(j), int(i))]].T
        off = bi != bj
        rowsum = np.zeros((nn, 3))
        np.add.at(rowsum, bi[off], np.abs(blocks[off]).sum(axis=2))
        for k in np.nonzero(~off)[0]:
            i = bi[k]
            s = 0.5 * (blocks[k] + blocks[k].T) * 0.1
            np.fill_diagonal(s, 0.0)
            blocks[k] = s + np.diag(1.05 * (rowsum[i] + np.abs(s).sum(axis=1)) + 1e-3)
    r = (3 * bi[:, None, None] + np.arange(3)[None, :, None]).repeat(3, axis=2)
    c = (3 * bj[:, None, None] + np.arange(3)[None, None, :]).repeat(3, axis=1)
    A = sp.csr_matrix((blocks.ravel(), (r.ravel(), c.ravel())), shape=(3 * nn, 3 * ncol_nodes))
    A.sort_indices()
    assert A.nnz == 9 * bi.size
    return A


def _near(i, count, nc, rng, reach=8):
    """`count` distinct column nodes within +-reach of node i (always including i when it exists)."""
    if count == 0:
        return np.zeros(0, np.int64)
    lo, hi = max(0, i - reach), min(nc, i + reach + 1)
    pool = np.setdiff1d(np.arange(lo, hi), [i])
    pick = rng.choice(pool, min(count - 1, pool.size), replace=False) if count > 1 else np.zeros(0, np.int64)
    return np.sort(np.concatenate([[i] if i < nc else [], pick]).astype(np.int64))


def _counts_to_matrix(counts, rng, ncol_nodes=None):
    nc = len(counts) if ncol_nodes is None else ncol_nodes
    return node_block([_near(i, int(c), nc, rng) for i, c in enumerate(counts)], nc, rng)


def nb_empty(seed=1, nn=3001, run=700):
    """Mixed counts 1..9 with empty nodes: the first two nodes, pairs of neighbours, a run of `run` nodes (longer than a
    1200-item tile: a tile starts inside it and one tile has no block at all) and the last three nodes.
    Returns (A, empty node indices)."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(1, 10, nn)
    empty = [0, 1, 400, 401, 1300, 1301, 1302] + list(range(1700, 1700 + run)) + [nn - 3, nn - 2, nn - 1]
    counts[empty] = 0
    return _counts_to_matrix(counts, rng), np.array(sorted(set(empty)))


def nb_singleton(seed=2, nn=2501):
    """Block diagonal: every node exactly one block, so NB == NN in every tile (the uniform path needs NB >= 2 NN)."""
    rng = np.random.default_rng(seed)
    return node_block([np.array([i]) for i in range(nn)], nn, rng)


def nb_mixed(seed=3, nn=3003):
    """A uniform stretch (5 blocks per node), random counts 1..12, then a uniform stretch of single blocks."""
    rng = np.random.default_rng(seed)
    t = nn // 3
    counts = np.concatenate([np.full(t, 5), rng.integers(1, 13, nn - 2 * t), np.full(t, 1)])
    return _counts_to_matrix(counts, rng)


def nb_small(nn, seed=4):
    """1, 2 or a few nodes (one tile; fewer tiles than resident CTAs)."""
    rng = np.random.default_rng(seed + nn)
    return _counts_to_matrix(rng.integers(1, min(nn, 5) + 1, nn), rng)


def nb_many(seed=5, nn=24001):
    """Enough nodes for thousands of 600-item tiles: every stage of every ring wraps many times."""
    rng = np.random.default_rng(seed)
    return _counts_to_matrix(rng.integers(1, 13, nn), rng)


def nb_banded(long_blocks, seed=6, nn=1201):
    """Tridiagonal node graph (3 blocks per node) except one node in the middle with `long_blocks` consecutive
    neighbour blocks: its rows are the longest, 3 * long_blocks non-zeros."""
    rng = np.random.default_rng(seed)
    m = nn // 2
    nbrs = [np.arange(max(0, i - 1), min(nn, i + 2)) for i in range(nn)]
    lo = m - long_blocks // 2
    nbrs[m] = np.arange(lo, lo + long_blocks)
    return node_block(nbrs, nn, rng)


def nb_rect(seed=7, nn=1501, nc=1709):
    """Rectangular node-block matrix (more column nodes than row nodes); SpMV only."""
    rng = np.random.default_rng(seed)
    return _counts_to_matrix(rng.integers(0, 11, nn), rng, ncol_nodes=nc)


def nb_spd(seed=8, nn=900, reach=4, p=0.6):
    """SPD node-block matrix for the solver: symmetric random band graph with its diagonal, no empty node."""
    rng = np.random.default_rng(seed)
    sets = [{i} for i in range(nn)]
    for i in range(nn):
        for j in range(i + 1, min(nn, i + reach + 1)):
            if rng.random() < p:
                sets[i].add(j); sets[j].add(i)
    return node_block([np.array(sorted(s)) for s in sets], nn, rng, spd=True)


# ----------------------------------------------------------------------------------------- row-group matrices
def _rows(lengths, ncols, rng, start=None):
    """CSR with the given row lengths; row r holds a run of consecutive columns from start[r] (wrapped)."""
    lengths = np.asarray(lengths, dtype=np.int64)
    n = lengths.size
    start = np.arange(n) if start is None else np.asarray(start)
    indptr = np.concatenate([[0], np.cumsum(lengths)])
    cols = np.concatenate([(s + np.arange(L)) % ncols for s, L in zip(start, lengths)]) if n else np.zeros(0)
    A = sp.csr_matrix((rng.standard_normal(int(indptr[-1])), cols.astype(np.int64), indptr), shape=(n, ncols))
    A.sort_indices()
    return A


def rg_lengths(lanes, seed=10, n=3000):
    """Row lengths 4 L - 1, 4 L, 4 L + 1 (one unrolled pass of the L-lane row loop -1/0/+1) mixed with 0, 1, L - 1, L,
    L + 1 and 8 L + 1."""
    rng = np.random.default_rng(seed + lanes)
    L = lanes
    menu = np.array([4 * L - 1, 4 * L, 4 * L + 1, 0, 1, L - 1, L, L + 1, 8 * L + 1])
    lengths = menu[rng.integers(0, menu.size, n)]
    lengths[: 3 * 50] = np.repeat([4 * L - 1, 4 * L, 4 * L + 1], 50)   # each edge length present in runs too
    return _rows(lengths, n + 8 * L + 2, rng)


def rg_empty_rows(seed=11, n=12000, run=5000):
    """Rows of 1..30 non-zeros with runs of empty rows: at the start, pairs in the middle, a run of `run` rows (more than
    two of the largest tiles, 2304 items, so tiles start inside it and one holds only empty rows) and at the end."""
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, 31, n)
    lengths[:3] = 0
    lengths[[1000, 1001, 2500, 2501, 2502]] = 0
    lengths[4000:4000 + run] = 0
    lengths[-4:] = 0
    return _rows(lengths, n + 40, rng, start=np.maximum(np.arange(n) - 15, 0))


def rg_long_rows(tile, seed=12, n=2500):
    """Rows longer than a tile of `tile` merge items: lengths tile + 1, 2 tile, and one of 3 tile + 200 (it spans more
    than 3 tiles), next to empty rows, among short rows."""
    rng = np.random.default_rng(seed)
    lengths = rng.integers(0, 20, n)
    lengths[[7, 1200, n - 1]] = [tile + 1, 2 * tile, 3 * tile + 200]
    lengths[[6, 8, 1199, 1201]] = 0
    return _rows(lengths, 3 * tile + 400, rng, start=np.minimum(np.arange(n), 150))


def rg_windows(seed=13, n=2000, per_row=48):
    """Columns 12 k + (r % 3): runs of three columns 9 apart, more than the 8-column gap the x windows merge, so every
    tile needs per_row (48 > 32) windows - the producers load the window descriptors in several rounds of 32."""
    rng = np.random.default_rng(seed)
    k = np.arange(per_row)
    cols = np.concatenate([12 * k + (r % 3) for r in range(n)])
    indptr = np.arange(n + 1) * per_row
    A = sp.csr_matrix((rng.standard_normal(cols.size), cols, indptr), shape=(n, 12 * per_row))
    A.sort_indices()
    return A


def rg_triples(lanes3, seed=14, n=1500):
    """Rows made of aligned triples of consecutive columns (the T3 index), with 2 L - 1, 2 L, 2 L + 1 triples per row
    (one pass of the two-triple unrolled loop -1/0/+1), 0, 1 and L triples."""
    rng = np.random.default_rng(seed + lanes3)
    L = lanes3
    menu = np.array([2 * L - 1, 2 * L, 2 * L + 1, 0, 1, L])
    trip = menu[rng.integers(0, menu.size, n)]
    trip[: 3 * 30] = np.repeat([2 * L - 1, 2 * L, 2 * L + 1], 30)
    nct = n + 2 * L + 2
    cols = [(3 * ((r + np.arange(t)) % nct))[:, None] + np.arange(3)[None, :] for r, t in enumerate(trip)]
    indptr = np.concatenate([[0], np.cumsum(3 * trip)])
    A = sp.csr_matrix((rng.standard_normal(int(indptr[-1])), np.concatenate([c.ravel() for c in cols]), indptr), shape=(n, 3 * nct))
    A.sort_indices()
    return A


# ----------------------------------------------------------------------------------------- invariants
def node_patterns_ok(A):
    """Rows 3n, 3n+1, 3n+2 share one column pattern made of aligned triples 3j, 3j+1, 3j+2."""
    A = sp.csr_matrix(A)
    if A.shape[0] % 3:
        return False
    ip, ix = A.indptr, A.indices
    for n in range(A.shape[0] // 3):
        r = [ix[ip[3 * n + k]:ip[3 * n + k + 1]] for k in range(3)]
        if not (np.array_equal(r[0], r[1]) and np.array_equal(r[0], r[2])) or r[0].size % 3:
            return False
        t = r[0].reshape(-1, 3)
        if np.any(t[:, 0] % 3) or np.any(t[:, 1] != t[:, 0] + 1) or np.any(t[:, 2] != t[:, 0] + 2):
            return False
    return True


def blocks_per_node(A):
    return np.diff(sp.csr_matrix(A).indptr)[0::3] // 3
