"""The rap multigrid hierarchy's host side (multigrid.HexMultigrid(coarse="rap"), rap_bytes, rap_setup_peak_bytes) without a
GPU: the ValueError refusals before any library call, the device bytes and set-up peak pinned from 16^3 to 512^3 and restated
from the level lists of gmg_cases and a direct count of the hex CSR's non-zeros, and the 512^3 voxel model fitting 80 GB."""
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


class _TwoRanks(_StubOperator):
    class comm:
        nranks, rank = 2, 0


@pytest.fixture
def no_library(monkeypatch):
    from pcg_mpi_solver_b200 import _lib

    def load():
        raise AssertionError("the library was loaded before the refusal")

    monkeypatch.setattr(_lib, "load", load)


def _block(ne=(8, 8, 8)):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    return HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0])


@pytest.mark.parametrize("op,ne,kw,match", [
    (_StubOperator, (8, 8, 8), dict(), "needs E_field"),
    (_StubOperator, (8, 8, 8), dict(coarsening="any"), "needs E_field"),
    (_StubOperator, (8, 8, 8), dict(E_field=np.ones((8, 8, 8)), coarsening="any"), "default coarsening"),
    (_TwoRanks, (8, 8, 8), dict(E_field=np.ones((8, 8, 8))), "one rank"),
    (_StubOperator, (4, 4, 4), dict(E_field=np.ones((4, 4, 4))), "at least 3 levels"),
    (_StubOperator, (8, 4, 8), dict(E_field=np.ones((8, 4, 8))), "at least 3 levels"),
    (_StubOperator, (9, 8, 8), dict(E_field=np.ones((8, 8, 9))), "does not coarsen"),
    (_StubOperator, (576, 576, 576), dict(E_field=np.ones((1, 1, 1))), "coarsest level has 2700 dofs"),
])
def test_refusals_come_before_any_library_call(no_library, op, ne, kw, match):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    with pytest.raises(ValueError, match=match):
        HexMultigrid(op(), _block(ne), coarse="rap", **kw)


def test_index_free_still_refuses_a_field(no_library):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    with pytest.raises(ValueError, match="E_field"):
        HexMultigrid(_StubOperator(), _block(), coarse="index_free", E_field=np.ones((8, 8, 8)))


def _nnz_by_count(ne):
    """Non-zeros of the clamped hex CSR counted node by node: 9 per (free node, free in-box neighbour) pair."""
    nx, ny, nz = ne
    total = 0
    for lz in range(nz + 1):
        cz = sum(1 for d in (-1, 0, 1) if 0 <= lz + d <= nz)
        for ly in range(ny + 1):
            cy = sum(1 for d in (-1, 0, 1) if 0 <= ly + d <= ny)
            for lx in range(1, nx + 1):
                total += 9 * cz * cy * sum(1 for d in (-1, 0, 1) if 1 <= lx + d <= nx)
    return total


@pytest.mark.parametrize("ne", [(2, 2, 2), (4, 2, 6), (8, 8, 8), (16, 4, 8), (5, 3, 7)])
def test_hex_csr_nnz_formula_against_a_count(ne):
    from pcg_mpi_solver_b200.multigrid import hex_csr_nnz
    assert hex_csr_nnz(ne) == _nnz_by_count(ne)


# (fine cube edge) -> (rap_bytes, rap_setup_peak_bytes)
PINNED = {16: (870508, 2654208), 32: (6656024, 21233664), 64: (51924036, 169869312), 128: (409957744, 1207959552),
          256: (3257698460, 2264924160), 512: (25973338056, 10871635968)}


def _restated(ne):
    lv = G.levels_of(ne)
    n = [3 * G.nfree(v) for v in lv]
    vectors = 8 * (5 * n[0] + 6 * sum(n[1:-1]) + 2 * n[-1] + n[-1] ** 2)
    csr = 0
    for l in range(2, len(lv) - 1):
        nnz = 9 * (3 * lv[l][0] - 2) * (3 * lv[l][1] + 1) * (3 * lv[l][2] + 1)
        csr += 12 * nnz + (4 if nnz < 2**31 - 1 else 8) * (n[l] + 1)
    el = [4608 * v[0] * v[1] * v[2] for v in lv]
    layer = 4608 * lv[1][0] * lv[1][1]
    layers = min(lv[1][2], max(2, 2 * ((1 << 30) // (2 * layer))))
    peak = el[2] + max(layers * layer, el[3] if len(lv) > 3 else 0)
    return vectors + csr, peak


@pytest.mark.parametrize("edge", sorted(PINNED))
def test_rap_bytes_and_setup_peak_pinned(edge):
    from pcg_mpi_solver_b200.multigrid import index_free_bytes, rap_bytes, rap_setup_peak_bytes
    ne = (edge,) * 3
    assert (rap_bytes(ne), rap_setup_peak_bytes(ne)) == _restated(ne) == PINNED[edge]
    assert rap_bytes(ne) > index_free_bytes(ne)


def test_slab_splits_128_into_two_and_512_into_pairs():
    """At 128^3 a level-1 layer is 64^2 elements (18.9 MB): the 1 GiB cap holds 56 of the 64 layers, so the set-up runs two
    slabs.  At 512^3 a layer is 302 MB: every slab is one pair of layers, and level 3 (1.2 GB) is the larger term."""
    layer = 4608 * 64 * 64
    assert (1 << 30) // layer == 56 and 56 < 64
    big = 4608 * 256 * 256
    assert (1 << 30) // big == 3 and 2 * big < 4608 * 64 ** 3


def test_rap_bytes_of_other_shapes_and_the_refusals():
    from pcg_mpi_solver_b200.multigrid import rap_bytes, rap_setup_peak_bytes
    assert (rap_bytes((16, 8, 12)), rap_setup_peak_bytes((16, 8, 12))) == _restated((16, 8, 12)) == (433152, 995328)
    for ne, match in (((4, 4, 4), "at least 3 levels"), ((9, 8, 8), "does not coarsen"), ((576,) * 3, "2700 dofs")):
        for f in (rap_bytes, rap_setup_peak_bytes):
            with pytest.raises(ValueError, match=match):
                f(ne)


def test_512_voxel_model_fits_an_80_gb_gpu():
    """The rap hierarchy (26.0 GB), the solver's five vectors and minv, b, x (8 fine vectors, 25.9 GB) and the fine Ck field
    (1.07 GB) take about 53 GB, under 80 GB; the set-up's element matrices (10.9 GB) are held before the CSR of level 2
    (6.1 GB) exists, so the set-up stays under 80 GB as well."""
    from pcg_mpi_solver_b200.multigrid import hex_csr_nnz, rap_bytes, rap_setup_peak_bytes
    ne = (512,) * 3
    n = 3 * G.nfree(ne)
    total = rap_bytes(ne) + 8 * n * 8 + 8 * 512 ** 3
    assert 52e9 <= total <= 54e9, total
    assert total + rap_setup_peak_bytes(ne) + 12 * hex_csr_nnz((128,) * 3) < 80e9
