"""The host restatement of HexMultigrid(coarsening="any") (tests/gmg_any_cases.py): the coarsening rule and its refusals,
the general P against the existing one on all-even boxes, the element-level Galerkin products with widths against P^T A P,
and pinned iteration counts of a host MG-PCG on odd and semi-coarsened boxes."""
import numpy as np
import pytest

from tests import gmg_any_cases as A
from tests import gmg_cases as G
from tests import voxel_cases as V


@pytest.mark.parametrize("ne", sorted(A.LEVELS))
def test_rule_levels(ne):
    from pcg_mpi_solver_b200.multigrid import any_levels
    assert A.levels(ne) == A.LEVELS[ne] == any_levels(ne)
    assert max(A.LEVELS[ne][-1]) <= 2


def test_rule_refusals():
    from pcg_mpi_solver_b200.multigrid import any_levels
    for ne in ((2, 2, 2), (1, 1, 1), (2, 1, 2)):
        for fn in (A.levels, any_levels):
            with pytest.raises(ValueError, match="coarsen"):
                fn(ne)
    big = (2 ** 33, 1, 1)        # 33 levels
    assert len(A.levels(big, max_levels=40)) == 33
    for fn in (A.levels, any_levels):
        with pytest.raises(ValueError, match="32 levels"):
            fn(big)
    assert len(any_levels((2 ** 31 - 1, 2, 2))) == 31     # the deepest box of int32 element counts


@pytest.mark.parametrize("nf", range(1, 12))
def test_positions_and_weights(nf):
    """s(0) = 0 and s(nc) = nf; gaps 1 or 2 with only the last gap of an odd axis 1 wide; every weight 0, 1/2 or 1; rows sum
    to 1."""
    s = A.positions(nf)
    assert s[0] == 0 and s[-1] == nf
    gaps = np.diff(s)
    if nf <= 2:
        assert np.all(gaps == 1)
    else:
        assert np.all(gaps[:-1] == 2) and gaps[-1] == (1 if nf % 2 else 2)
    P = A.interp_1d(s)
    assert set(np.unique(P)) <= {0.0, 0.5, 1.0}
    assert np.all(P.sum(axis=1) == 1.0)
    assert np.all(P[s, np.arange(len(s))] == 1.0)


@pytest.mark.parametrize("ne", [(4, 4, 4), (8, 8, 8), (16, 8, 12), (8, 4, 6), (24, 16, 8)])
def test_general_P_equals_existing_on_even_boxes(ne):
    assert abs(A.prolongation_any(ne) - G.prolongation_matrix(ne)).max() == 0


@pytest.mark.parametrize("ne", [(5, 4, 3), (7, 3, 9), (1, 5, 9), (3, 3, 3), (16, 16, 15), (8, 8, 5), (25, 17, 9), (38, 4, 16)])
@pytest.mark.parametrize("kind", ["random", "constant"])
def test_galerkin_restatement_equals_ptap(ne, kind):
    """Every level assembled from the element-level Galerkin products with widths equals scipy P^T A P to 1e-13 of its
    largest entry, for a random field and for a constant one."""
    f = V.random_field(ne, seed=sum(ne)) if kind == "random" else np.full((ne[2], ne[1], ne[0]), 2.5)
    for l, (M, Q) in enumerate(zip(A.level_matrices(f, 0.5), A.ptap_matrices(f, 0.5))):
        assert M.shape == Q.shape
        assert abs(M - Q).max() <= 1e-13 * abs(Q).max(), l


def test_galerkin_even_box_equals_voxel_restatement():
    """On an all-even box the widths are all 2 and the products are voxel_cases.galerkin's."""
    f = V.random_field((8, 4, 6), seed=3)
    for a, b in zip(A.level_elements(f, 0.5), V.level_elements(f, 0.5)):
        assert np.array_equal(a, b)


# (box, contrast) -> host MG-PCG iterations to 1e-8 (degree 2, lo 0.25, load of hexmesh.load_vector, h = 1 / ne[0]); contrast
# 100 is gmg_any_cases.field_of's inclusion field
PINNED = {((16, 16, 15), 1): 12, ((16, 16, 15), 100): 47, ((15, 15, 15), 1): 13, ((15, 15, 15), 100): 49,
          ((17, 17, 17), 1): 20, ((17, 17, 17), 100): 58, ((25, 17, 9), 1): 26, ((25, 17, 9), 100): 69,
          ((38, 4, 16), 1): 18, ((38, 4, 16), 100): 127, ((8, 8, 5), 1): 12, ((8, 8, 5), 100): 33}


@pytest.mark.parametrize("ne,contrast", sorted(PINNED))
def test_host_mg_pcg_iterations(ne, contrast):
    it = A.host_pcg_iters(ne, contrast)
    assert abs(it - PINNED[(ne, contrast)]) <= 2, it
    assert it < 500
