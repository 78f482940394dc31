"""The voxel-model multigrid across ranks without a GPU: the host restatement of tests/voxel_dd_cases.py against the one-rank
field hierarchy (voxel_cases.HostFieldMultigrid), the refusals of HexMultigrid(op, block, blocks=..., E_field=...) before
any library call, and the cap on the gathered element matrices."""
import numpy as np
import pytest

from tests import gmg_dd_cases as D
from tests import voxel_cases as V
from tests import voxel_dd_cases as VD

GRIDS = [((2, 1, 1), 8), ((3, 1, 1), 8), ((2, 2, 1), 8), ((2, 2, 2), 8), ((2, 1, 1), 16)]


def _field(kind, ng):
    return V.random_field(ng, seed=5) if kind == "random" else V.two_phase(ng, 100.0, seed=3, radii=(1.0, 3.0))


@pytest.mark.parametrize("kind", ["random", "two_phase"])
@pytest.mark.parametrize("pgrid,per", GRIDS)
def test_host_ranked_field_hierarchy_matches_the_one_rank_one(pgrid, per, kind):
    boxes = D.grid_boxes(pgrid, per)
    levels, why = D.coarsen(boxes)
    assert why is None
    la = len(levels) - 1
    ng = boxes[0].ng
    h = boxes[0].h
    field = _field(kind, ng)
    glob = V.level_elements(field, h)
    host = V.HostFieldMultigrid(field, h)
    ranked = VD.HostRankFieldMultigrid(levels, field, h, host.lam)
    # every rank's element matrices are the one-rank ones of the same elements, bit for bit
    for l in range(la + 1):
        for b, k in zip(levels[l], ranked.kel[l]):
            assert np.array_equal(k, VD.box_slice(glob[l], b))
    # the gather gives the one-rank matrices of level la, so the replicated levels are the one-rank levels
    assert np.array_equal(ranked.gathered, glob[la])
    for k, A in enumerate(ranked.sub.mats):
        ref = host.mats[la + k]
        assert (A != ref).nnz == 0
    # ranked levels: interior rows equal, the exchange-added product the global one's to rounding
    rng = np.random.default_rng(11)
    for l in range(1, la):
        Ag = host.mats[l]
        x = rng.standard_normal(Ag.shape[0])
        y = Ag @ x
        got = D.exchange(levels[l], [a @ x[b.global_dofs()] for a, b in zip(ranked.A[l], levels[l])])
        for b, v in zip(levels[l], got):
            assert np.max(np.abs(v - y[b.global_dofs()])) <= 1e-14 * np.max(np.abs(y))
    # the distributed V-cycle
    r = rng.standard_normal(host.A[0].n)
    want = host.apply(r)
    z = ranked.apply(D.to_local(levels[0], r))
    for b, v in zip(levels[0], z):
        w = want[b.global_dofs()]
        assert np.linalg.norm(v - w) <= 1e-13 * np.linalg.norm(w)


def test_interior_rows_of_a_ranked_level_are_the_global_rows():
    """Rows of nodes inside a rank's box (no other rank holds them) sum the same element matrices as the global row."""
    boxes = D.grid_boxes((2, 2, 1), 8)
    levels, _ = D.coarsen(boxes)
    field = _field("random", boxes[0].ng)
    host = V.HostFieldMultigrid(field, boxes[0].h)
    ranked = VD.HostRankFieldMultigrid(levels, field, boxes[0].h, host.lam)
    l = 1
    for r, (b, A) in enumerate(zip(levels[l], ranked.A[l])):
        nbr, lists, _ = D.lists(levels[l], r)
        shared = np.zeros(b.n, dtype=bool)
        for li in lists:
            shared[li] = True
        gd = b.global_dofs()
        Ag = host.mats[l][gd][:, gd]
        inner = np.flatnonzero(~shared)
        assert inner.size > 0
        assert np.allclose((A[inner] - Ag[inner]).toarray(), 0.0, rtol=0, atol=1e-13 * abs(Ag).max())


class _StubRanks:
    """Stands in for a multi-rank SubdomainOperator: every refusal must come before the operator or the library is used."""
    device = "cpu"

    def __init__(self, n, rank=0, nranks=2):
        self.n = n
        self.comm = type("C", (), {"nranks": nranks, "rank": rank})()

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


def _split(ng=(16, 8, 8), pgrid=(2, 1, 1)):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, partition_blocks
    h = 1.0 / ng[0]
    return [HexBlock(b.ng, b.e0, b.ne, h=h) for b in partition_blocks(ng, pgrid)]


def _refused(blocks, field, match, rank=0, **kw):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    with pytest.raises(ValueError, match=match):
        HexMultigrid(_StubRanks(blocks[rank].n, rank, len(blocks)), blocks[rank], blocks=blocks, E_field=field, **kw)


@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("bad", [float("nan"), 0.0, -1.0, float("inf"), -float("inf")])
def test_a_bad_value_anywhere_in_the_global_field_is_refused_on_every_rank(no_library, rank, bad):
    """The bad value lies in rank 1's box; rank 0 refuses it as well, before any collective step."""
    import torch
    blocks = _split()
    f = V.random_field(blocks[0].ng, seed=2)
    f[5, 4, 12] = bad
    _refused(blocks, f, "finite and positive", rank)
    _refused(blocks, torch.from_numpy(f), "finite and positive", rank)


def test_wrong_fields_are_refused(no_library):
    from pcg_mpi_solver_b200.hexmesh import block_field
    blocks = _split()
    f = V.random_field(blocks[0].ng, seed=2)
    _refused(blocks, block_field(f, blocks[0]), "shape")           # a rank's slice, as generate_matrix takes it
    _refused(blocks, f[:, :, :-1], "shape")
    _refused(blocks, f.astype(np.float32), "float64")
    _refused(blocks, f.tolist(), "numpy array or a torch tensor")


def test_other_refusals_stay(no_library):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blocks = _split()
    f = V.random_field(blocks[0].ng, seed=2)
    _refused(blocks, f, "E_field", coarse="index_free")
    _refused(blocks, f, "coarsening", coarsening="any")
    with pytest.raises(ValueError, match="needs `blocks`"):
        HexMultigrid(_StubRanks(blocks[0].n), blocks[0], E_field=f)
    with pytest.raises(ValueError, match="blocks\\[comm.rank\\]"):
        HexMultigrid(_StubRanks(blocks[0].n), blocks[0], blocks=blocks[::-1], E_field=f)
    with pytest.raises(ValueError, match="does not coarsen"):     # rank_levels' refusals come first
        odd = _split((18, 8, 8))
        HexMultigrid(_StubRanks(odd[0].n), odd[0], blocks=odd, E_field=V.random_field(odd[0].ng, seed=2))


def _two_boxes(ng, x_cut):
    """Two ranks split at x = x_cut (even), so that the halved cut is odd and la = 1."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    h = 1.0 / ng[0]
    return [HexBlock(ng, (0, 0, 0), (x_cut, ng[1], ng[2]), h=h), HexBlock(ng, (x_cut, 0, 0), (ng[0] - x_cut, ng[1], ng[2]), h=h)]


def test_cap_on_the_gathered_element_matrices():
    from pcg_mpi_solver_b200.hexmesh import partition_blocks
    from pcg_mpi_solver_b200.multigrid import MAX_GATHERED_ELEMENTS, gathered_elements, rank_levels
    assert MAX_GATHERED_ELEMENTS == 4096 and MAX_GATHERED_ELEMENTS * 576 * 8 == 18874368    # 18.9 MB of matrices
    # the bench's weak-scaled stacks: 8 ranks of 128^3 gather 4^3 elements, of 160^3 10^3
    assert gathered_elements(rank_levels(partition_blocks((256,) * 3, (2, 2, 2)))) == 64
    assert gathered_elements(rank_levels(partition_blocks((320,) * 3, (2, 2, 2)))) == 1000
    assert gathered_elements(rank_levels(_two_boxes((32, 32, 32), 18))) == 4096
    lv = rank_levels(_two_boxes((64, 32, 32), 34))
    assert len(lv) == 2 and lv[-1][0].ng == (32, 16, 16)
    with pytest.raises(ValueError, match="8192 elements"):
        gathered_elements(lv)


def test_the_cap_is_a_refusal_before_any_library_call(no_library):
    blocks = _two_boxes((64, 32, 32), 34)
    f = V.random_field(blocks[0].ng, seed=2)
    for rank in (0, 1):
        _refused(blocks, f, "8192 elements", rank)


def test_an_accepted_field_reaches_the_operator(no_library):
    """At the cap (4096 gathered elements) and with a valid field the constructor goes on to op.jacobi()."""
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blocks = _two_boxes((32, 32, 32), 18)
    f = V.random_field(blocks[0].ng, seed=2)
    with pytest.raises(AssertionError, match="jacobi"):
        HexMultigrid(_StubRanks(blocks[1].n, 1), blocks[1], blocks=blocks, E_field=f)
