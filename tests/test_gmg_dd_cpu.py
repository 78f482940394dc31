"""The multigrid hierarchy across ranks on the host (tests/gmg_dd_cases.py): coarsening rule, gathered level and refusals
(also those of multigrid.rank_levels, which the library's constructor uses), the global boxes against the one-rank
hierarchy, per-level lists and ownership against hexmesh.interface_lists, the owner-weighted restriction, the distributed
Lanczos estimate and the whole distributed V-cycle against gmg_cases.HostMultigrid."""
import numpy as np
import pytest

from tests import gmg_cases as G
from tests import gmg_dd_cases as D

GRIDS = [((1, 1, 1), 8), ((2, 1, 1), 8), ((3, 1, 1), 8), ((2, 2, 1), 8), ((2, 2, 2), 4), ((2, 2, 2), 8), ((2, 1, 1), 16)]


def _hexblocks(boxes):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    return [HexBlock(b.ng, b.e0, b.ne, h=b.h) for b in boxes]


@pytest.mark.parametrize("pgrid,per", GRIDS)
def test_levels_and_global_boxes(pgrid, per):
    from pcg_mpi_solver_b200.hexmesh import partition_blocks
    from pcg_mpi_solver_b200.multigrid import rank_levels
    boxes = D.grid_boxes(pgrid, per)
    ng = boxes[0].ng
    assert [(b.e0, b.ne) for b in boxes] == [(tuple(b.e0), tuple(b.ne)) for b in partition_blocks(ng, pgrid)]
    levels, why = D.coarsen(boxes)
    assert why is None
    la = len(levels) - 1
    assert la == int(np.log2(per)) - 1          # per, per/2, ..., 2 on every rank
    assert D.global_boxes(levels) == G.levels_of(ng)
    lib_levels = rank_levels(_hexblocks(boxes))
    assert [[(b.ng, b.e0, b.ne) for b in lv] for lv in lib_levels] == [[(b.ng, b.e0, b.ne) for b in lv] for lv in levels]


def test_refusals():
    from pcg_mpi_solver_b200.multigrid import rank_levels
    cases = {
        "coarsen": D.grid_boxes((2, 1, 1), 2),                                                    # la = 0
        "tile": D.grid_boxes((2, 1, 1), 8)[:1] + [D.Box((16, 8, 8), (6, 0, 0), (10, 8, 8))],       # overlap
        "gathered": [D.Box((100, 100, 100), (0, 0, 0), (50, 100, 100)), D.Box((100, 100, 100), (50, 0, 0), (50, 100, 100))],
        "coarse": [D.Box((12, 18, 18), (0, 0, 0), (6, 18, 18)), D.Box((12, 18, 18), (6, 0, 0), (6, 18, 18))],
    }
    hole = D.grid_boxes((2, 1, 1), 8)[:1]
    cases["tile_gap"] = [D.Box((16, 8, 8), b.e0, b.ne) for b in hole]
    odd_e0 = [D.Box((12, 8, 8), (0, 0, 0), (6, 8, 8)), D.Box((12, 8, 8), (6, 0, 0), (6, 8, 8))]   # e0 = 6 -> 3 after one halving
    levels, why = D.coarsen(odd_e0)
    assert why is None and len(levels) == 2            # halved once (e0 6 -> 3), then stops on the odd e0 and ne
    for name, boxes in cases.items():
        levels, why = D.coarsen(boxes)
        assert why == name.split("_")[0], name
        with pytest.raises(ValueError):
            rank_levels(_hexblocks(boxes))


@pytest.mark.parametrize("pgrid,per", GRIDS)
def test_lists_weights_and_ownership(pgrid, per):
    from pcg_mpi_solver_b200.hexmesh import interface_lists
    levels, _ = D.coarsen(D.grid_boxes(pgrid, per))
    for lv in levels:
        hb = _hexblocks(lv)
        count = np.zeros(3 * D.nfree(lv[0].ng))
        for r, b in enumerate(lv):
            nbr, lists, w = D.lists(lv, r)
            nbr2, lists2, w2 = interface_lists(hb, r)
            assert nbr == nbr2 and all(np.array_equal(a, c) for a, c in zip(lists, lists2)) and np.array_equal(w, w2)
            np.add.at(count, b.global_dofs(), w)
        assert np.all(count == 1.0)                 # every global dof owned exactly once


@pytest.mark.parametrize("pgrid,per", [((2, 1, 1), 8), ((3, 1, 1), 8), ((2, 2, 1), 8), ((2, 2, 2), 8)])
def test_restriction_across_ranks(pgrid, per):
    levels, _ = D.coarsen(D.grid_boxes(pgrid, per))
    rng = np.random.default_rng(per + len(levels[0]))
    for l in range(len(levels) - 1):
        ng = levels[l][0].ng
        rf = rng.standard_normal(3 * D.nfree(ng))
        P = G.prolongation_matrix(ng)
        want, mag = P.T @ rf, abs(P).T @ np.abs(rf)
        got = D.restrict_ranks(levels, l, D.to_local(levels[l], rf))
        for b, v in zip(levels[l + 1], got):   # <= 27 terms per rank's partial, then <= 8 partials
            assert np.all(np.abs(v - want[b.global_dofs()]) <= (27 + 8) * 2.0 ** -53 * mag[b.global_dofs()])
        # without the weights an interface node is counted once per rank that holds it
        bad = D.restrict_ranks(levels, l, D.to_local(levels[l], rf), weighted=False)
        assert max(np.abs(v - want[b.global_dofs()]).max() for b, v in zip(levels[l + 1], bad)) > 1e-3


@pytest.mark.parametrize("pgrid,per", [((2, 1, 1), 8), ((3, 1, 1), 8), ((2, 2, 1), 8), ((2, 2, 2), 4)])
def test_vcycle_and_lambda_across_ranks(pgrid, per):
    boxes = D.grid_boxes(pgrid, per)
    levels, _ = D.coarsen(boxes)
    ng, h = boxes[0].ng, boxes[0].h
    one = G.HostMultigrid(ng, h)
    for l in range(len(levels) - 1):
        dinv = [1.0 / d for d in D.exchange(levels[l], [b.csr().diagonal() for b in levels[l]])]
        lam = D.lanczos_ranks(levels[l], dinv)
        assert abs(lam - one.lam[l]) <= 1e-10 * one.lam[l], (l, lam, one.lam[l])
    dd = D.HostRankMultigrid(levels, h, one.lam)
    r = np.random.default_rng(11).standard_normal(3 * D.nfree(ng))
    want = one.apply(r)
    got = dd.apply(D.to_local(levels[0], r))
    for b, z in zip(levels[0], got):
        assert np.linalg.norm(z - want[b.global_dofs()]) <= 1e-13 * np.linalg.norm(want)
