"""The synthetic interface plans of tests/halo_cases.py and their host reference, checked without a GPU: `expected` equals
the oracle's exchange (oracle/ref_pcg.py exchange_add, pcg_solver.py:303-334) bit for bit, the cases reach the kernel
edges they are built for, and the plan-level refusals agree with what pcgb_halo_create refuses."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import halo_cases as H


def _ys(p, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(n) * 2.0 ** rng.integers(-30, 31, n) for n in p["n"]]


@pytest.mark.parametrize("name", list(H.CASES))
def test_expected_matches_oracle_exchange(name):
    p = H.plan(name)
    parts = [R.CsrPart(sp.identity(p["n"][r], format="csr"), np.zeros(p["n"][r]), p["nbr"][r], p["lists"][r], part_id=r)
             for r in range(p["world"])]
    for seed in range(2):
        ys = _ys(p, seed)
        want = H.expected(ys, p)
        got = R.exchange_add(parts, [y.copy() for y in ys])
        for r in range(p["world"]):
            assert np.array_equal(want[r].view(np.uint64), got[r].view(np.uint64)), (name, r)
            assert H.refusal(p, r) is None


def test_expected_pins_list_order():
    """Cancelling copies: the sum depends on the neighbour order, and `expected` follows the list order, not rank order."""
    p = H.make_plan(3, {(0, 1): 1, (0, 2): 1, (1, 2): 1}, hubs=(0, 1, 2))
    assert p["nbr"][0] == [2, 1]
    ys = [np.zeros(n) for n in p["n"]]
    ys[0][p["lists"][0][0][0]] = 1.0
    ys[2][p["lists"][2][p["nbr"][2].index(0)][0]] = 2.0 ** 53
    ys[1][p["lists"][1][p["nbr"][1].index(0)][0]] = -(2.0 ** 53)
    got = H.expected(ys, p)[0][p["lists"][0][0][0]]
    assert got == (1.0 + 2.0 ** 53) - 2.0 ** 53 == 0.0      # list order 2, 1; rank order 1, 2 would give 1.0


def test_cases_reach_the_kernel_edges():
    def ms(name):
        p = H.plan(name)
        return [H.m_of(p, r) for r in range(p["world"])], [H.ndof_of(p, r) for r in range(p["world"])], p

    m, nd, p = ms("w2_one")
    assert m == [1, 1]
    m, nd, p = ms("w2_1025")
    assert m == [H.PACK_PER_CTA + 1] * 2
    m, nd, p = ms("w3_pack_edge")
    assert m == [H.PACK_PER_CTA - 1, H.PACK_PER_CTA, H.PACK_PER_CTA + 1]
    assert [H.max_multiplicity(p, r) for r in range(3)] == [2, 2, 2]
    m, nd, p = ms("w3_unpack_edge")
    assert nd == [H.UNPACK_PER_CTA - 1, H.UNPACK_PER_CTA, H.UNPACK_PER_CTA + 1] and m == [400, 300, 300]
    m, nd, p = ms("w3_stride")
    assert m == [160, 160, 200]
    # the rank with the larger m stores first into both others' buffers: even with its own m as the parity stride its
    # stores stay inside their 2 * m receive entries
    for s in (0, 1):
        assert p["nbr"][s][0] == 2 and 0 + m[2] + len(p["lists"][s][0]) <= 2 * m[s]
    m, nd, p = ms("w3_empty")
    assert m == [0, 300, 300] and p["nbr"][0] == [1] and len(p["lists"][0][0]) == 0
    assert len(p["lists"][1][p["nbr"][1].index(0)]) == 0
    m, nd, p = ms("w4_big")
    assert m[0] == H.BIG_M and -(-m[0] // H.PACK_PER_CTA) == 193 and m[0] >= 100 * min(m)
    assert H.max_multiplicity(p, 0) == 3 and nd[0] == m[0] - 2
    m, nd, p = ms("w4_mixed")
    assert m[0] == 4097 and m[3] == 0 and p["nbr"][3] == []
    m, nd, p = ms("w4_hub")
    assert [H.max_multiplicity(p, r) for r in range(4)] == [3, 3, 3, 3]
    # list order is never ascending where a rank has two or more neighbours
    multi = 0
    for name in H.CASES:
        p = H.plan(name)
        for r in range(p["world"]):
            if len(p["nbr"][r]) >= 2:
                multi += 1
                assert p["nbr"][r] != sorted(p["nbr"][r]), (name, r)
    assert multi >= 10
    # lists are distinct within themselves, pairs have equal lengths
    for name in H.CASES:
        p = H.plan(name)
        for r in range(p["world"]):
            for j, s in enumerate(p["nbr"][r]):
                assert len(np.unique(p["lists"][r][j])) == len(p["lists"][r][j])
                assert len(p["lists"][s][p["nbr"][s].index(r)]) == len(p["lists"][r][j])
    assert sorted({H.CASES[k][0] for k in H.CASES}) == [2, 3, 4]


def test_refused_plans_are_refused_on_the_host():
    expect = {"duplicate_neighbour": "listed twice", "duplicate_index": "appears twice", "neighbour_self": "bad neighbour table",
              "neighbour_negative": "bad neighbour table", "neighbour_nranks": "bad neighbour table",
              "index_out_of_range": "out of range", "index_negative": "out of range"}
    bad = H.refused_plans()
    assert set(bad) == set(expect)
    for name, (nbr, lists, n) in bad.items():
        p = {"world": 4, "n": [n], "nbr": [nbr], "lists": [lists]}
        assert H.refusal(p, 0, nranks=4) == expect[name], name
    # an empty list is not a refusal: it is dropped
    assert H.refusal(H.plan("w3_empty"), 0) is None
