"""The multi-rank rap hierarchy's host side (HexMultigrid(op, block, blocks=..., E_field=..., coarse="rap"), rap_rank_bytes)
without a GPU: every refusal, old and new, raised before any library call on every rank alike, and the per-rank device bytes
pinned on several splits and restated level by level from rank_levels and hex_csr_nnz."""
import numpy as np
import pytest

from tests import voxel_cases as V


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


def _split(ng, pgrid):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, partition_blocks
    h = 1.0 / ng[0]
    return [HexBlock(b.ng, b.e0, b.ne, h=h) for b in partition_blocks(ng, pgrid)]


def _x_tiling(ng, cuts):
    """Boxes of the whole y and z extent, cut along x at the given widths."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    out, x = [], 0
    for w in cuts:
        out.append(HexBlock(ng, (x, 0, 0), (w, ng[1], ng[2]), h=1.0 / ng[0]))
        x += w
    return out


def _make(blocks, rank, field, **kw):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    return HexMultigrid(_StubRanks(blocks[rank].n, rank, len(blocks)), blocks[rank], blocks=blocks, E_field=field, coarse="rap", **kw)


def _refused_on_every_rank(blocks, field, match, **kw):
    for rank in range(len(blocks)):
        with pytest.raises(ValueError, match=match):
            _make(blocks, rank, field, **kw)


# splits whose rank boxes halve only once (la = 1): level 1 would be the gathered level
LA1 = [((12, 6, 6), None, "2x1x1 of 6^3: the halved boxes are 3 wide"),
       ((32, 16, 16), (18, 14), "an x cut at 18: the halved cut 9 is odd")]


@pytest.mark.parametrize("ng,cuts,what", LA1)
def test_la_1_splits_are_refused_on_every_rank(no_library, ng, cuts, what):
    from pcg_mpi_solver_b200.multigrid import rank_levels
    blocks = _x_tiling(ng, cuts) if cuts else _split(ng, (2, 1, 1))
    assert len(rank_levels(blocks)) == 2, what
    _refused_on_every_rank(blocks, V.random_field(blocks[0].ng, seed=2), "halve at least twice")


def test_the_existing_field_refusals_come_first(no_library):
    """rank_levels, check_global_field and gathered_elements refuse before the rap rule, on every rank alike."""
    from pcg_mpi_solver_b200.hexmesh import block_field
    blocks = _split((32, 16, 16), (2, 1, 1))
    f = V.random_field(blocks[0].ng, seed=2)
    fnan = f.copy()
    fnan[-1, -1, -1] = float("nan")           # in the last rank's part
    _refused_on_every_rank(blocks, fnan, "finite and positive")
    _refused_on_every_rank(blocks, block_field(f, blocks[0]), "shape")
    _refused_on_every_rank(blocks, f.astype(np.float32), "float64")
    odd = _split((18, 8, 8), (2, 1, 1))       # the fine level does not coarsen
    _refused_on_every_rank(odd, V.random_field(odd[0].ng, seed=2), "does not coarsen")
    big = _x_tiling((64, 32, 32), (34, 30))   # la = 1 and 8192 gathered elements: the cap fires first
    _refused_on_every_rank(big, V.random_field(big[0].ng, seed=2), "8192 elements")


def test_the_one_rank_rap_refusals_stay(no_library):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blocks = _split((32, 16, 16), (2, 1, 1))
    f = V.random_field(blocks[0].ng, seed=2)
    with pytest.raises(ValueError, match="needs E_field"):
        _make(blocks, 0, None)
    with pytest.raises(ValueError, match="default coarsening"):
        _make(blocks, 1, f, coarsening="any")
    with pytest.raises(ValueError, match="needs `blocks`"):
        HexMultigrid(_StubRanks(blocks[0].n), blocks[0], E_field=f, coarse="rap")
    with pytest.raises(ValueError, match="blocks\\[comm.rank\\]"):
        HexMultigrid(_StubRanks(blocks[0].n), blocks[0], blocks=blocks[::-1], E_field=f, coarse="rap")


@pytest.mark.parametrize("pgrid", [(2, 1, 1), (3, 1, 1), (2, 2, 1), (2, 2, 2)])
def test_an_accepted_split_reaches_the_operator(no_library, pgrid):
    """With la >= 2 and a valid field every rank goes on to op.jacobi(), the first step after the refusals."""
    blocks = _split(tuple(16 * p for p in pgrid), pgrid)
    f = V.random_field(blocks[0].ng, seed=2)
    for rank in range(len(blocks)):
        with pytest.raises(AssertionError, match="jacobi"):
            _make(blocks, rank, f)


def _nnz_by_count(ne, x_lo):
    """Non-zeros of a box's sub-assembled hex CSR counted node by node: 9 per (free node, free in-box neighbour) pair."""
    nx, ny, nz = ne
    total = 0
    for lz in range(nz + 1):
        cz = sum(1 for d in (-1, 0, 1) if 0 <= lz + d <= nz)
        for ly in range(ny + 1):
            cy = sum(1 for d in (-1, 0, 1) if 0 <= ly + d <= ny)
            for lx in range(x_lo, nx + 1):
                total += 9 * cz * cy * sum(1 for d in (-1, 0, 1) if x_lo <= lx + d <= nx)
    return total


@pytest.mark.parametrize("ne", [(2, 2, 2), (4, 2, 6), (8, 8, 8), (5, 3, 7)])
@pytest.mark.parametrize("x_lo", [0, 1])
def test_hex_csr_nnz_of_rank_boxes_against_a_count(ne, x_lo):
    from pcg_mpi_solver_b200.multigrid import hex_csr_nnz
    assert hex_csr_nnz(ne, x_lo) == _nnz_by_count(ne, x_lo)


def _restated(levels, rank):
    """What mg_build allocates on `rank`, level by level, in bytes."""
    from pcg_mpi_solver_b200.multigrid import hex_csr_nnz

    def csr(ne, n, x_lo):
        nnz = hex_csr_nnz(ne, x_lo)
        return 12 * nnz + (4 if nnz < 2**31 - 1 else 8) * (n + 1)

    la = len(levels) - 1
    total = 0
    for l in range(la + 1):
        b = levels[l][rank]
        total += 8 * b.n                                    # ownership weights
        if l == 0:
            total += 8 * 5 * b.n                            # z, r, d, q, D^-1
        elif l < la:
            total += 8 * 6 * b.n + (csr(b.ne, b.n, b.x_lo) if l >= 2 else 0)   # b, x, r, d, q, D^-1 (+ CSR from level 2)
        else:
            total += 8 * 2 * b.n                            # gathered: b, x
    ne = tuple(levels[-1][0].ng)
    rep = [ne]
    while all(v % 2 == 0 and v >= 4 for v in rep[-1]):
        rep.append(tuple(v // 2 for v in rep[-1]))
    for k, v in enumerate(rep):
        n = 3 * v[0] * (v[1] + 1) * (v[2] + 1)
        total += 8 * (2 * n + n * n) if k == len(rep) - 1 else 8 * 6 * n + csr(v, n, 1)
    return total


# name -> (ng, pgrid, x cuts); WANT: rap_rank_bytes of every rank (the ranks off x = 0 hold one more x plane per level)
PINNED = {
    "2x1x1 of 8^3": ((16, 8, 8), (2, 1, 1), None),
    "2x1x1 of 16^3": ((32, 16, 16), (2, 1, 1), None),
    "3x1x1 of 16^3": ((48, 16, 16), (3, 1, 1), None),
    "2x2x1 of 16^3": ((32, 32, 16), (2, 2, 1), None),
    "2x2x2 of 16^3": ((32, 32, 32), (2, 2, 2), None),
    "x tiling 24 + 8": ((32, 16, 16), None, (24, 8)),
    "2x2x2 of 64^3": ((128, 128, 128), (2, 2, 2), None),
    "2x1x1 of 256^3": ((512, 256, 256), (2, 1, 1), None),
}
WANT = {
    "2x1x1 of 8^3": [206448, 222960],
    "2x1x1 of 16^3": [1071580, 1186708],
    "3x1x1 of 16^3": [1189084, 1304212, 1304212],
    "2x2x1 of 16^3": [1238620, 1353748, 1238620, 1353748],
    "2x2x2 of 16^3": [1198856, 1313984] * 4,
    "x tiling 24 + 8": [1700668, 975772],
    "2x2x2 of 64^3": [59578336, 61476616] * 4,
    "2x1x1 of 256^3": [3722151692, 3751639076],
}


@pytest.mark.parametrize("name", sorted(PINNED))
def test_rap_rank_bytes_pinned_and_restated(name):
    from pcg_mpi_solver_b200.multigrid import rank_levels, rap_rank_bytes
    ng, pgrid, cuts = PINNED[name]
    blocks = _x_tiling(ng, cuts) if cuts else _split(ng, pgrid)
    levels = rank_levels(blocks)
    assert len(levels) >= 3
    got = [rap_rank_bytes(levels, r) for r in range(len(blocks))]
    assert got == [_restated(levels, r) for r in range(len(blocks))]
    assert got == WANT[name]


def test_x_tiling_24_8_has_level_1_widths_off_the_brick():
    """The hand-built tiling's level-1 boxes are 12 and 4 elements wide: neither free-node count is a multiple of k_mg_rap1's
    8-node x brick (12 on the clamped box, 5 on the other), and the second box has a free low-x face."""
    from pcg_mpi_solver_b200.multigrid import rank_levels
    lv = rank_levels(_x_tiling((32, 16, 16), (24, 8)))
    assert [b.ne[0] for b in lv[1]] == [12, 4] and [b.x_lo for b in lv[1]] == [1, 0]
    assert [(b.ne[0] + 1 - b.x_lo) % 8 for b in lv[1]] == [4, 5]
    assert len(lv) - 1 == 2


def test_rap_rank_bytes_without_a_level_1_matrix():
    """Against the ranked field hierarchy's bytes (its level-1 CSR included), rap saves exactly the level-1 CSR per rank."""
    from pcg_mpi_solver_b200.multigrid import hex_csr_nnz, rank_levels, rap_rank_bytes
    levels = rank_levels(_split((64, 32, 32), (2, 1, 1)))
    for r in range(2):
        b = levels[1][r]
        nnz = hex_csr_nnz(b.ne, b.x_lo)
        assert _restated(levels, r) == rap_rank_bytes(levels, r)
        assert 12 * nnz + 4 * (b.n + 1) > rap_rank_bytes(levels, r) // 4
    with pytest.raises(ValueError, match="halve at least twice"):
        rap_rank_bytes(rank_levels(_split((12, 6, 6), (2, 1, 1))), 0)
