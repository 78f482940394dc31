"""CPU checks of the SpMV edge-case generators (tests/spmv_cases.py): each case has the shape its GPU test relies on."""
import numpy as np
import pytest
import scipy.sparse as sp

from tests import spmv_cases as C

NODE = {
    "empty": lambda: C.nb_empty()[0], "singleton": C.nb_singleton, "mixed": C.nb_mixed, "1-node": lambda: C.nb_small(1),
    "2-nodes": lambda: C.nb_small(2), "1-tile": lambda: C.nb_small(40), "many": C.nb_many, "rect": C.nb_rect,
    "banded": lambda: C.nb_banded(225), "spd": C.nb_spd,
}


@pytest.mark.parametrize("name", sorted(NODE))
def test_node_block_rows_share_aligned_triples(name):
    A = NODE[name]()
    assert C.node_patterns_ok(A) and A.nnz % 9 == 0 and A.has_sorted_indices
    assert C.node_patterns_ok(sp.csr_matrix(np.ones((3, 6)))) and not C.node_patterns_ok(sp.csr_matrix(np.eye(3)))


def test_node_block_counts():
    A, empty = C.nb_empty()
    bpn = C.blocks_per_node(A)
    assert np.array_equal(np.nonzero(bpn == 0)[0], empty)
    assert bpn[0] == bpn[1] == 0 and bpn[-1] == 0 and bpn[400] == bpn[401] == 0 and bpn.max() == 9
    # with 1200-item tiles a tile starts inside the run of 700 empty nodes and one tile has no block at all
    s = C.tile_row_starts(A.indptr, 1200, 3)
    assert (bpn[s[1:-1] // 3] == 0).any()
    assert any(s[b + 1] > s[b] and A.indptr[s[b + 1]] == A.indptr[s[b]] for b in range(len(s) - 1))
    assert np.all(C.blocks_per_node(C.nb_singleton()) == 1)
    m = C.blocks_per_node(C.nb_mixed())
    assert np.all(m[:1001] == 5) and np.all(m[-1001:] == 1) and set(m[1001:-1001]) == set(range(1, 13))
    assert C.nb_small(1).shape == (3, 3) and C.nb_small(2).shape == (6, 6)
    R = C.nb_rect()
    assert R.shape == (3 * 1501, 3 * 1709) and (C.blocks_per_node(R) == 0).any()
    # the value tail: nnz not a multiple of 8 (nnz / 9 blocks not a multiple of 8) on these cases
    for name in ("empty", "mixed", "1-node", "2-nodes", "1-tile", "rect"):
        assert (NODE[name]().nnz // 9) % 8 != 0, name


@pytest.mark.parametrize("inplace", [1, 0])
def test_banded_longest_node_at_the_limit(inplace):
    limit = C.BSR_MAX_ROW[inplace]
    # spmv.cuh build_plan_t: default tile (6100 | 4608) - 3 (max_row + 1) must hold two nodes of 3 (max_row + 1) items
    base = 6100 if inplace else 4608
    assert base - 3 * (limit + 1) >= 6 * (limit + 1) and base - 3 * (limit + 2) < 6 * (limit + 2)
    for blocks in (limit // 3, limit // 3 + 1):
        A = C.nb_banded(blocks)
        lens = np.diff(A.indptr)
        assert lens.max() == 3 * blocks and np.count_nonzero(lens == lens.max()) == 3
        long_node = int(np.argmax(lens)) // 3
        cols = A.indices[A.indptr[3 * long_node]:A.indptr[3 * long_node + 1]]
        assert np.all(np.diff(cols) == 1)                 # consecutive neighbour columns: one x window
    assert 3 * (limit // 3) <= limit < 3 * (limit // 3 + 1)


def test_spd_case_is_spd():
    A = C.nb_spd()
    assert abs(A - A.T).max() == 0
    assert (C.blocks_per_node(A) > 0).all()
    assert np.linalg.eigvalsh(A.toarray()).min() > 0


@pytest.mark.parametrize("lanes", [4, 8, 16, 32])
def test_row_lengths_at_the_lane_edges(lanes):
    lens = np.diff(C.rg_lengths(lanes).indptr)
    for L in (4 * lanes - 1, 4 * lanes, 4 * lanes + 1, 0):
        assert (lens == L).sum() >= 50, L
    T = C.rg_triples(lanes)
    tri = np.diff(T.indptr)
    assert np.all(tri % 3 == 0)
    for t in (2 * lanes - 1, 2 * lanes, 2 * lanes + 1, 0):
        assert (tri == 3 * t).sum() >= 30, t
    c = T.indices.reshape(-1, 3)
    assert np.all(c[:, 0] % 3 == 0) and np.all(c[:, 1] == c[:, 0] + 1) and np.all(c[:, 2] == c[:, 0] + 2)


def test_row_group_cases():
    E = C.rg_empty_rows()
    lens = np.diff(E.indptr)
    assert lens[:3].sum() == 0 and lens[-4:].sum() == 0 and lens[4000:9000].sum() == 0 and (lens[9000:] > 0).any()
    for tile in (512, 1024, 1536, 1920, 2304):    # the row-group tile sizes: one tile holds only empty rows
        s = C.tile_row_starts(E.indptr, tile)
        assert (lens[s[1:-1]] == 0).any()
        assert any(s[b + 1] > s[b] and E.indptr[s[b + 1]] == E.indptr[s[b]] for b in range(len(s) - 1)), tile
    for tile in (256, 1024):
        L = np.diff(C.rg_long_rows(tile).indptr)
        assert L.max() == 3 * tile + 200 and (L > tile).sum() == 3 and L[6] == L[8] == 0
    W = C.rg_windows()
    row = W.indices[W.indptr[0]:W.indptr[1]]
    assert row.size == 48 and np.all(np.diff(row) > 9)  # 48 runs, gaps above the 8-column merge gap: > 32 windows per tile


def test_reference_product_and_tile_starts():
    rng = np.random.default_rng(0)
    A = sp.random(50, 40, density=0.1, random_state=1, format="csr")
    A = sp.vstack([sp.csr_matrix((3, 40)), A, sp.csr_matrix((2, 40))]).tocsr()   # empty rows at both ends
    x = rng.standard_normal(40)
    y, scale = C.ref_spmv(A, x)
    assert y.dtype == np.longdouble and np.allclose(np.asarray(y, dtype=float), A @ x, rtol=1e-15, atol=1e-15)
    assert np.all(y[:3] == 0) and np.all(y[-2:] == 0) and np.allclose(scale, abs(A) @ np.abs(x))
    # merge-path partition: every tile covers about tile_items rows + non-zeros; unit 3 snaps to nodes
    ip = A.indptr
    s = C.tile_row_starts(ip, 16, 1)
    assert s[0] == 0 and s[-1] == A.shape[0] and np.all(np.diff(s) >= 0)
    items = np.diff(s) + np.diff(ip[s])
    assert items[:-1].max() <= 16 + A.getnnz(axis=1).max()
    assert np.all(C.tile_row_starts(ip, 16, 3)[:-1] % 3 == 0)
