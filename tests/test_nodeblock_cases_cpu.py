"""CPU checks of the node-block restatements in tests/nodeblock_cases.py: the fp64 row order against an exact rational fma
and the long-double product, the order pin against every wrong order, the run stream on hand-built chains and the ring
choice on worked examples."""
import numpy as np
import pytest

from tests import nodeblock_cases as N
from tests import spmv_cases as C


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


# ------------------------------------------------------------------------------------------------ rows_f64
def test_fma_exact_rounding_and_zero_signs():
    u = 1.0 + 2.0 ** -30
    assert N.fma_exact(u, u, -(1.0 + 2.0 ** -29)) == 2.0 ** -60          # the product is not rounded
    assert N.fma_exact(2.0 ** 53, 1.0, 1.0) == 2.0 ** 53                   # ties to even
    assert N.fma_exact(2.0 ** 53, 1.0, 3.0) == 2.0 ** 53 + 4.0
    for a, b, c, neg in [(-0.0, 1.0, -0.0, True), (0.0, 1.0, -0.0, False), (-0.0, -1.0, -0.0, False), (-0.0, 1.0, 0.0, False),
                         (1.0, 1.0, -1.0, False), (-1.0, 1.0, 1.0, False)]:
        r = N.fma_exact(a, b, c)
        assert r == 0.0 and (np.signbit(r) == neg), (a, b, c, r)


@pytest.mark.parametrize("case", ["nb-mixed", "nb-empty", "nb-rect", "order-pin"])
def test_rows_f64_matches_the_rational_fma_and_long_double(case):
    if case == "order-pin":
        A, x, _ = N.order_pin()
    else:
        A = {"nb-mixed": C.nb_mixed, "nb-empty": lambda: C.nb_empty()[0], "nb-rect": C.nb_rect}[case]().tocsr()
        x = N.signed_x(A.shape[1], seed=len(case))
    y = N.rows_f64(A, x)
    rng = np.random.default_rng(3)
    rows = np.unique(np.concatenate([[0, A.shape[0] - 1], rng.integers(0, A.shape[0], 400)]))
    assert np.array_equal(_bits(y[rows]), _bits(N.rows_reference(A, x, rows)))
    assert np.array_equal(_bits(N.rows_f64(A, x, rows)), _bits(y[rows]))         # sampled sub-CSR
    if case != "order-pin":
        ref, scale = C.ref_spmv(A, x)
        err = np.abs(y.astype(np.longdouble) - ref)
        k = np.diff(A.indptr)
        assert np.all(err <= (k + 2) * N.EPS * scale + 1e-300)


def test_rows_f64_empty_rows_are_positive_zero():
    A, empty = C.nb_empty()
    y = N.rows_f64(A, N.signed_x(A.shape[1], seed=1))
    rows = np.concatenate([3 * empty, 3 * empty + 1, 3 * empty + 2])
    assert np.all(y[rows] == 0.0) and not np.signbit(y[rows]).any()


def test_exact_dot():
    rng = np.random.default_rng(0)
    x, y = N.signed_x(5000, seed=2), rng.standard_normal(5000)
    d, s = N.exact_dot(x, y)
    from fractions import Fraction
    assert d == float(sum(Fraction(a) * Fraction(b) for a, b in zip(x.tolist(), y.tolist())))
    assert s == pytest.approx(float(np.abs(x * y).sum()), rel=1e-12)


# ------------------------------------------------------------------------------------------------ order pin
def test_order_pin_separates_every_wrong_order():
    A, x, kinds = N.order_pin()
    y = N.rows_f64(A, x)
    assert set(kinds) == set(N.ORDER_KINDS)
    node = np.repeat(np.arange(kinds.size), 3)
    wrong = {"nest": dict(nest="rev"), "nofma": dict(nest="nofma"), "order": dict(order="rev"), "start": dict(start=-0.0)}
    catch = {"nest": {"nest", "nofma"}, "nofma": {"nofma"}, "order": {"order-a", "order-b"}, "start": {"negzero", "empty"}}
    for name, kw in wrong.items():
        w = N.rows_reference(A, x, **kw)
        diff = _bits(w) != _bits(y)
        assert diff.any(), name
        for k in catch[name]:                         # every row of the kind tells the orders apart
            assert diff[kinds[node] == k].all(), (name, k)
    # the documented bits of each kind
    u = 1.0 + 2.0 ** -30
    for k, want in [("order-a", 0.0), ("order-b", 0.0), ("nofma", 2.0 ** -60), ("negzero", 0.0), ("empty", 0.0)]:
        got = y[kinds[node] == k]
        assert np.array_equal(_bits(got), _bits(np.full(got.size, want))), k
    nest = y[kinds[node] == "nest"]
    assert np.all(nest == (u + u) + u)


# ------------------------------------------------------------------------------------------------ run stream
def _chain(nn, reach=(-1, 0, 1), ids=None):
    rng = np.random.default_rng(0)
    nbrs = [np.array([i + r for r in reach if 0 <= i + r < nn]) for i in range(nn)]
    A = C.node_block(nbrs, nn, rng)
    pos = N._block_positions(A)
    dic = rng.standard_normal((len(reach) + 3, 9))
    vid = np.concatenate([np.array([r for r in range(len(reach)) if 0 <= i + reach[r] < nn]) + (ids or {}).get(i, 0)
                          for i in range(nn)])
    A.data[pos] = dic[vid]
    return A


def test_vd_runs_one_chain():
    """Nodes 1..nn-2 repeat their predecessor (node 1 joins node 0 only if both have three blocks: node 0 has two)."""
    A = _chain(20)
    segs, words, cov = N.vd_runs(A, [0, 20])
    # node 0 (2 blocks): explicit; node 1 heads a run through node 18; node 19 (2 blocks): explicit
    assert segs == [[(0, False), (1, True), (19, False)]]
    assert cov.tolist() == [18]
    assert words.tolist() == [1 + 2 * 3 + 2 + 3 + 2]
    # cut into tiles: runs restart at every tile start
    segs, words, cov = N.vd_runs(A, [0, 5, 6, 12, 20])
    assert segs == [[(0, False), (1, True)], [(0, False)], [(0, True)], [(0, True), (7, False)]]
    assert cov.tolist() == [4, 0, 6, 7]
    assert words.tolist() == [1 + 4 + 2 + 3, 1 + 2 + 3, 1 + 2 + 3, 1 + 4 + 3 + 2]
    assert N.stream_words(words) == (int(words.sum()), 12)   # tile 0: words 0..9 -> aligned window 0..12


def test_vd_runs_breaks_and_segment_cap():
    """Runs of two (the id changes every other node): 2 segments per pair; more than 8 segments -> one explicit segment."""
    nn = 40
    A = _chain(nn, ids={i: 3 * ((i // 2) % 2) for i in range(nn)})
    join, nb = N.node_joins(A)
    assert join[3:nn - 1:2].all() and not join[2:nn - 1:2].any()   # node 2k + 1 joins node 2k, node 2k does not join
    segs, words, cov = N.vd_runs(A, [0, 8, 24, nn])
    assert segs[0] == [(0, False), (2, True), (4, True), (6, True)] and cov[0] == 6   # node 1 (3 blocks) does not join node 0 (2)
    assert segs[1] == [(2 * k, True) for k in range(8)] and cov[1] == 16                # 8 pairs: exactly the cap
    assert words[1] == 1 + 2 * 8 + 3 * 8
    uncapped = N.vd_runs(A, [0, 8, 26, nn], cap=10 ** 9)
    capped = N.vd_runs(A, [0, 8, 26, nn])
    assert len(uncapped[0][1]) == 9 and uncapped[2][1] == 18                          # 9 pairs: one over the cap
    assert capped[0][1] == [(0, False)] and capped[2][1] == 0 and capped[1][1] == 3 + nb[8:26].sum()
    segs, words, cov = N.vd_runs(A, [0, 0, nn])
    assert segs[0] == [] and words[0] == 1 and cov[0] == 0                             # an empty tile: the header only


def test_vd_runs_empty_nodes_join():
    """Empty nodes have as many blocks as an empty predecessor and no block that differs: they join its run."""
    A, empty = C.nb_empty()
    join, nb = N.node_joins(A)
    e = np.asarray(empty)
    pairs = e[np.isin(e - 1, e)]
    assert join[pairs].all()
    starts = C.tile_row_starts(A.indptr, 1200, unit=3) // 3
    segs, words, cov = N.vd_runs(A, starts)
    assert N.expected_run_nodes(A, 1200) == cov.sum() > 0
    assert words.sum() == sum(1 + 2 * len(s) for s in segs) + sum(
        int(nb[s0 + f]) if run else int(nb[s0 + f:s0 + (sg[k + 1][0] if k + 1 < len(sg) else s1 - s0)].sum())
        for sg, s0, s1 in zip(segs, starts[:-1], starts[1:]) for k, (f, run) in enumerate(sg))


# ------------------------------------------------------------------------------------------------ ring
def test_producers():
    assert [N.producers(s) for s in range(1, 17)] == [1, 2, 3, 4, 1, 2, 1, 4, 1, 2, 1, 4, 1, 2, 1, 4]


def test_vd_ring_worked_examples():
    # hex 128^3 default plan, with the caps the plan reports (x_cap 732, cap_nodes 56, cap_words 100, D = 96, 2 CTAs per
    # SM): 14 stages do not fit two CTAs, 12 do - CW 6: G = 6; CW 8: G = 8; CW 12: no G >= 10 fits, G = 9 (DESIGN)
    for cw, g, smem in [(6, 6, 105216), (8, 8, 110592), (12, 9, 113280)]:
        r = N.vd_ring(cap_x=732, cap_nodes=56, cap_words=100, vd=96, cw=cw, ctas_per_sm=2)
        assert r["stage_bytes"] == (732 * 8 + 58 * 8 + 100 * 4 + 32 + 127) & ~127 == 6784
        assert (r["stages"], r["group"], r["producers"], r["smem"]) == (12, g, 4, smem), r
        assert N.SMEM_SM // (r["smem"] + 2 * 6784 + 2048) == 1                        # two more stages: one CTA per SM
    # a small plan: the deepest ring for each CW (2 G + 2, at most 16)
    for cw, s in [(6, 14), (8, 16), (12, 16)]:
        r = N.vd_ring(cap_x=64, cap_nodes=8, cap_words=40, vd=10, cw=cw, ctas_per_sm=2)
        assert (r["stages"], r["group"]) == (s, cw)
    # a large dictionary: G + 2 stages for CW 6, and G < CW for CW 12
    r = N.vd_ring(cap_x=300, cap_nodes=30, cap_words=300, vd=900, cw=6, ctas_per_sm=2)
    assert (r["stages"], r["group"], r["producers"]) == (8, 6, 4), r
    r = N.vd_ring(cap_x=300, cap_nodes=30, cap_words=300, vd=900, cw=12, ctas_per_sm=2)
    assert r["group"] < 12 and r["stages"] == r["group"] + 2, r
    # forced rings: the request, clamped to 16, G = min(CW, stages)
    for env, s, g, p in [(1, 1, 1, 1), (3, 3, 3, 3), (5, 5, 5, 1), (6, 6, 6, 2), (7, 7, 6, 1), (10, 10, 6, 2), (14, 14, 6, 2),
                         (16, 16, 6, 4), (17, 16, 6, 4)]:
        r = N.vd_ring(cap_x=64, cap_nodes=8, cap_words=40, vd=10, cw=6, ctas_per_sm=2, env_stages=env)
        assert (r["stages"], r["group"], r["producers"]) == (s, g, p), env
    assert N.vd_ring(cap_x=6000, cap_nodes=200, cap_words=3000, vd=1024, cw=12, ctas_per_sm=1, env_stages=16) is None


def test_vd_ring_default_search_order():
    """Walk a dictionary size up: the ring gets shallower by even steps down to G + 2, then G drops below CW."""
    seen = []
    for vd in range(1, 2000, 7):
        r = N.vd_ring(cap_x=300, cap_nodes=30, cap_words=300, vd=vd, cw=8, ctas_per_sm=2)
        if r is None:
            break
        seen.append((r["group"], r["stages"]))
    assert seen[0] == (8, 16)
    assert (8, 10) in seen and any(g < 8 for g, _ in seen)
    assert all(s % 2 == 0 and g + 2 <= s <= min(2 * g + 2, 16) for g, s in seen)
    assert seen == sorted(seen, reverse=True)       # never deeper or wider as the dictionary grows
