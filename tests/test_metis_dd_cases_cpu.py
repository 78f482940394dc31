"""The subdomain builder's interface tables on the element splits of tests/metis_dd_cases.py, and on concrete's golden
8-way split when data/concrete.zip is staged: symmetric neighbour tables, positional list pairs on the full and the free
lists, 0/1 owner weights of the lowest id summing to n_global_eff, multiplicities equal to the number of parts that hold
a node; and each split reaches the case it is there for. The exact exchange of the workers is pinned against a plain
per-dof restatement."""
import json
import os

import numpy as np
import pytest

from tests import metis_dd_cases as C


@pytest.mark.parametrize("name", list(C.CASES))
def test_builder_tables(name):
    _, ep, subs = C.subdomains(name)
    assert len(subs) == C.CASES[name][1] and np.bincount(ep, minlength=len(subs)).min() > 0
    assert C.table_failures(subs) == []


def test_cases_reach_what_they_are_for():
    f = {name: C.features(C.subdomains(name)[2]) for name in C.CASES}
    assert all(v["empty_free_lists"] == 0 for v in f.values())           # impossible on a hex model (module docstring)
    for name in ("metis2", "metis3", "metis4"):
        assert f[name]["max_multiplicity"] == C.CASES[name][1]
    # random8: disconnected parts, each neighbours every other, and a node in all 8 parts
    assert f["random8"]["max_multiplicity"] == 8 and f["random8"]["all_neighbours"]
    ng = C.CASES["random8"][0]
    ep = C.elepart("random8")
    assert all(C.connected_components(ng, ep, p) > 1 for p in range(8))
    # hand: an edge-only pair, a node-only pair (a 3-dof list), a one-element part with clamped shared nodes
    _, ep, subs = C.subdomains("hand")
    assert f["hand"]["min_free_list"] == 3 and f["hand"]["min_elements"] == 1
    p0, p3 = subs[0], subs[3]
    lens = dict(zip(p0.nbr, (len(v) for v in p0.ovrlp)))
    assert lens[1] == 9 and lens[2] == 3                                   # 3 nodes on the edge, 1 node
    assert p3.nbr == [4] and len(p3.ovrlp_full[0]) == 21 and len(p3.ovrlp[0]) == 12


def _plain_exchange(tables, ys):
    """One dof at a time: y[i] + copy of neighbour 0 + copy of neighbour 1 + ... as Python floats."""
    out = []
    for r, (_, nbr, lists) in enumerate(tables):
        y = [float(v) for v in ys[r]]
        for j, s in enumerate(nbr):
            theirs = tables[s][2][tables[s][1].index(r)]
            for t, i in enumerate(lists[j]):
                y[int(i)] += float(ys[s][int(theirs[t])])
        out.append(np.array(y))
    return out


@pytest.mark.parametrize("name", ["metis3", "random8", "hand"])
def test_exchange_is_the_plain_per_dof_sum(name):
    """C.exchange, the workers' expected halo result, adds in the order the peer and NCCL unpack kernels document."""
    _, _, subs = C.subdomains(name)
    tables = [(s.id, s.nbr, s.ovrlp) for s in subs]
    rng = np.random.default_rng(5)
    ys = [rng.standard_normal(s.n) * 2.0 ** rng.integers(-40, 41, s.n) for s in subs]
    got = C.exchange(tables, ys)
    want = _plain_exchange(tables, ys)
    assert all(C.same_bits(g, w) for g, w in zip(got, want))
    # a consistent vector's exchanged local products are consistent: the gathered copies agree with the global product
    m, _, hsubs = C.subdomains(name, assemble=True)
    v = [C.probe(s.dof_eff_global) for s in hsubs]
    y = C.exchange(tables, [s.A @ x for s, x in zip(hsubs, v)])
    from pcg_mpi_solver_b200.partition import build_subdomains
    one = build_subdomains(m, np.zeros(m.n_elem, dtype=np.int64), 1)[0]
    assert np.array_equal(one.dof_eff_global, m.dof_eff)
    K = one.A
    yg = K @ C.probe(m.dof_eff)
    pos = {int(g): k for k, g in enumerate(m.dof_eff)}
    for s, ys_ in zip(hsubs, y):
        idx = np.array([pos[int(g)] for g in s.dof_eff_global])
        bound = np.abs(K[idx]) @ np.abs(C.probe(m.dof_eff))
        assert np.all(np.abs(ys_ - yg[idx]) <= 1e-13 * bound)


@pytest.mark.skipif(not os.path.exists(C.CONCRETE_ZIP), reason="data/concrete.zip not staged")
def test_concrete_golden_split_tables(record_property):
    """The golden 8-way split of concrete (the reference's own partition): the same guarantees, the reference's neighbour
    tables (part 7 has 7 neighbours), several pattern groups and sign flips per part. Whether any free list is empty is
    reported: concrete is the model where it can happen."""
    from pcg_mpi_solver_b200.partition import partition_mesh
    g = json.load(open(os.path.join(C.GOLD, "concrete_ref.json")))
    ep = np.load(os.path.join(C.GOLD, "concrete_elepart_8.npy")).astype(np.int64)
    subs = partition_mesh(C.CONCRETE_ZIP, 8, elepart=ep, assemble=False)
    assert C.table_failures(subs) == []
    assert [s.nbr for s in subs] == [g["runs"]["8"]["parts"][str(k)]["nbrs"] for k in range(8)]
    f = C.features(subs)
    assert f["max_neighbours"] == 7 == len(subs[7].nbr)
    assert all(len(s.groups) > 1 and any(gr.sign.any() for gr in s.groups) for s in subs)
    record_property("concrete_empty_free_lists", f["empty_free_lists"])
    print(f"concrete 8-way: {f['empty_free_lists']} empty free lists, max multiplicity {f['max_multiplicity']}")
