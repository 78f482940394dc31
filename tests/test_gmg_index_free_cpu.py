"""The index-free multigrid hierarchy's host side (multigrid.HexMultigrid(coarse="index_free"), index_free_bytes) without a
GPU: the ValueError refusals before any library call, the device bytes of the hierarchy pinned, and the level lists of the
default coarsening from 16^3 to 640^3."""
import numpy as np
import pytest

from tests import gmg_cases as G


class _StubOperator:
    """Stands in for a SubdomainOperator: every refusal must come before the operator or the library is used."""
    n = 3 * 8 * 9 * 9
    device = "cpu"
    comm = None

    def jacobi(self):
        raise AssertionError("jacobi() called before the refusal")

    @property
    def _solver(self):
        raise AssertionError("the solver handle was used before the refusal")


@pytest.fixture
def no_library(monkeypatch):
    from pcg_mpi_solver_b200 import _lib

    def load():
        raise AssertionError("the library was loaded before the refusal")

    monkeypatch.setattr(_lib, "load", load)


def _block(ne=(8, 8, 8)):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    return HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0])


@pytest.mark.parametrize("kw,match", [
    (dict(coarse="index_free", E_field=np.ones((8, 8, 8))), "E_field"),
    (dict(coarse="index_free", coarsening="any"), "coarsening"),
    (dict(coarse="index_free", coarsening="any", E_field=np.ones((8, 8, 8))), "coarsening"),
    (dict(coarse="dense"), "coarse must be"),
    (dict(coarse="CSR"), "coarse must be"),
    (dict(coarse=None), "coarse must be"),
])
def test_refusals_come_before_any_library_call(no_library, kw, match):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    with pytest.raises(ValueError, match=match):
        HexMultigrid(_StubOperator(), _block(), **kw)


def _nfree_dofs(ne):
    return 3 * G.nfree(ne)


# (fine cube edge) -> (coarsest cube edge, levels, bytes of pcgb_mg_info): 512 is the largest power-of-two cube the rule
# accepts under 1536 coarsest dofs; 576 ends at 9^3 (2700 dofs) and is refused; 640 ends at 5^3 and is accepted
LEVELS = {16: (2, 4, 686784), 32: (2, 5, 4979520), 64: (2, 6, 38263872), 128: (2, 7, 300359232), 256: (2, 8, 2380505664),
          384: (3, 8, 8009396640), 448: (7, 7, 12721484832), 512: (2, 9, 18955414080), 640: (5, 8, 36990060960)}


@pytest.mark.parametrize("edge", sorted(LEVELS))
def test_level_lists_and_bytes_of_the_index_free_hierarchy(edge):
    """index_free_bytes = 8 (5 n_0 + 6 sum n_l over the smoothed coarse levels + 2 n_c + n_c^2), restated here from the
    level list of gmg_cases (the host oracle's coarsening), and pinned."""
    from pcg_mpi_solver_b200.multigrid import index_free_bytes
    ne = (edge,) * 3
    lv = G.levels_of(ne)
    coarsest, nlev, pinned = LEVELS[edge]
    assert lv[-1] == (coarsest,) * 3 and len(lv) == nlev
    assert [v[0] for v in lv] == [edge >> l for l in range(nlev)]
    n = [_nfree_dofs(v) for v in lv]
    assert n[-1] <= 1536
    formula = 8 * (5 * n[0] + 6 * sum(n[1:-1]) + 2 * n[-1] + n[-1] ** 2)
    assert index_free_bytes(ne) == formula == pinned


def test_index_free_bytes_at_512_fit_an_80_gb_gpu_with_the_solver():
    """18.96 GB of hierarchy plus the solver's five vectors (16.2 GB) and minv, b, x: about 45 GB at 512^3; 640^3 needs
    about 88 GB."""
    from pcg_mpi_solver_b200.multigrid import index_free_bytes
    for edge, lo, hi in ((512, 44e9, 46e9), (640, 87e9, 90e9)):
        n = _nfree_dofs((edge,) * 3)
        total = index_free_bytes((edge,) * 3) + 8 * n * (5 + 3)
        assert lo <= total <= hi, (edge, total)


@pytest.mark.parametrize("ne,match", [((576, 576, 576), "coarsest level has 2700 dofs"), ((9, 8, 8), "does not coarsen"),
                                      ((2, 8, 8), "does not coarsen")])
def test_index_free_bytes_refuses_what_create_refuses(ne, match):
    from pcg_mpi_solver_b200.multigrid import index_free_bytes
    with pytest.raises(ValueError, match=match):
        index_free_bytes(ne)
