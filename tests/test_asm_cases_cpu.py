"""The device-assembly cases of tests/asm_cases.py reach the kernel edges they are built for (no GPU needed)."""
import numpy as np
import pytest

from tests import asm_cases as C


def _distinct(sub):
    rows, indptr = C.ref_rows(sub)[:2]
    return np.diff(indptr)


@pytest.mark.parametrize("nd", C.PATTERN_SIZES)
def test_pattern_cases(nd):
    for variant in C.PATTERN_VARIANTS:
        sub = C.pattern_case(nd, variant)
        (g,) = sub.groups
        assert g.loc_dof.shape[0] == nd and g.ck.size >= 2
        assert all(np.unique(g.loc_dof[:, e]).size == nd for e in range(g.ck.size))
        cand = C.candidates(sub)
        assert cand.max() <= C.MAX_CAND and cand.max() >= 2 * nd           # rows shared by several elements
        frac = g.sign.mean()
        assert {"plain": frac == 0, "signs20": 0.1 < frac < 0.3 or nd * g.ck.size < 40 and 0 < frac < 1,
                "signsall": frac == 1, "ck4": frac == 0, "clamped": frac == 0}[variant], (variant, frac)
        if variant == "ck4":
            assert g.ck.max() / g.ck.min() > 1e3
        free = np.isin(g.loc_dof, sub.loc_dof_eff)
        if variant == "clamped":
            assert not free[:, -1].any()                                     # one element touches no free dof
            touched = np.unique(g.loc_dof[:, :-1])
            assert 0.05 <= 1 - np.isin(touched, sub.loc_dof_eff).mean() <= 0.2
        else:
            assert free.all()


@pytest.mark.parametrize("total", [2047, 2048, 2049])
def test_candidate_cases(total):
    assert C.candidates(C.candidate_case(total)).max() == total


def test_bitonic_case():
    sub = C.bitonic_case()
    cand, dist = C.candidates(sub), _distinct(sub)
    got = set(zip(cand[sub.extra["centres"]].tolist(), dist[sub.extra["centres"]].tolist()))
    assert got == set(C.bitonic_stars())
    assert set(C.BITONIC_TOTALS) <= set(cand.tolist())
    for m in range(1, 33):
        assert {32 * m - 1, 32 * m, 32 * m + 1} <= set(dist.tolist()), m
    assert cand.max() <= C.MAX_CAND


def test_structure_case():
    sub = C.structure_case()
    pos = np.full(sub.ndof, -1)
    pos[sub.loc_dof_eff] = np.arange(sub.n)
    cand, dist = C.candidates(sub), _distinct(sub)
    assert (cand[pos[sub.extra["empty"]]] == 0).all() and pos[sub.extra["empty"]].tolist() == [0, pos[260], sub.n - 1]
    assert (dist[pos[sub.extra["lonely"]]] == 1).all() and (cand[pos[sub.extra["lonely"]]] > 1).all()
    nes = [g.ck.size for g in sub.groups]
    assert nes[0] > 0 and nes[-1] == 0 and any(nes[k] == 0 and nes[k - 1] > 0 and nes[k + 1] > 0 for k in range(1, len(nes) - 1))
    hub = pos[sub.extra["hub"]]
    assert cand[hub] == 2000 and max(g.loc_dof.shape[0] for g in sub.groups if g.ck.size) <= 10
    assert sum((g.loc_dof == sub.extra["hub"]).sum() for g in sub.groups) == 200
    assert cand.max() <= C.MAX_CAND
    sub0 = C.no_rows_case()
    assert sub0.n == 0 and sub0.groups[0].ck.size > 0


def test_key_field_cases():
    sub = C.many_groups_case()
    assert len(sub.groups) == C.GROUPS_300 and {g.loc_dof.shape for g in sub.groups} == {(4, 3)}
    low = np.zeros(sub.ndof, bool)
    high = np.zeros(sub.ndof, bool)
    for k, g in enumerate(sub.groups):
        (high if k >= 256 else low)[g.loc_dof.ravel()] = True
    assert (low & high).sum() > 100                                          # rows mix groups on both sides of 256
    sub = C.wide_pattern_case()
    assert sub.groups[0].loc_dof.shape[0] == 255 and C.candidates(sub).max() <= C.MAX_CAND


def test_many_elements_case():
    sub = C.many_elements_case()
    (g,) = sub.groups
    assert g.loc_dof.shape == (1, C.BIG_NE) and C.BIG_NE > 2**24
    per_dof = np.bincount(g.loc_dof[0], minlength=sub.ndof)
    assert per_dof.max() <= 20 and np.ptp(g.ck) > 0.5
    assert (g.loc_dof[0, 2**24:] != g.loc_dof[0, :C.BIG_NE - 2**24]).all()    # element e and e - 2^24 sit on different dofs


@pytest.mark.parametrize("n", C.SCAN_SIZES)
def test_scan_cases(n):
    sub = C.scan_case(n)
    assert sub.n == n
    lens = np.diff(C.ref_rows(sub)[1]) if n < 2**20 else None
    cand = C.candidates(sub)
    blocks = np.add.reduceat(cand, np.arange(0, n, 1024))
    assert (blocks > 0).all() and np.unique(blocks).size > min(blocks.size - 1, 2)   # every 1024-row block carries a different sum
    if lens is not None:
        assert lens.min() == 0 and lens.max() >= 10


def test_order_case_discriminates():
    sub = C.order_case()
    doc, fill, rev = (C.ordered_sums(sub, o) for o in ("documented", "fill", "reversed"))
    for r in sub.extra["rows"]:
        assert doc[(r, r)] == 0.0 and fill[(r, r)] == 1.0 and rev[(r, r)] == 1.0
    for g in sub.groups:                                                   # every product exact: Ke integers, Ck powers of two
        assert np.array_equal(g.ke, np.round(g.ke)) and np.all(np.log2(g.ck) == np.round(np.log2(g.ck)))


def test_duplicate_case():
    sub = C.duplicate_case()
    (g,) = sub.groups
    free = np.isin(g.loc_dof, sub.loc_dof_eff)
    same = lambda a, b: (g.loc_dof[a] == g.loc_dof[b]) & free[a]
    assert same(3, 10).sum() >= 10 and same(5, 38).sum() >= 10 and (same(1, 2) & same(1, 33)).sum() >= 5
    assert all(np.unique(g.loc_dof[:, e]).size == C.DUP_ND for e in range(50, 60))


def test_band_case_row_lengths():
    for ne in (1, 2, 5):
        assert np.array_equal(np.diff(C.ref_rows(C.band_case(ne))[1]), C.band_row_lengths(ne))
    assert C.band_row_lengths(C.INT64_NE).sum() >= 2**31


def test_reference_matches_host_assembly():
    from pcg_mpi_solver_b200.partition import _assemble
    for sub in (C.pattern_case(33, "clamped"), C.duplicate_case(), C.structure_case(), C.spd_case()):
        K = _assemble(sub.groups, sub.ndof)
        A = K[sub.loc_dof_eff][:, sub.loc_dof_eff].tocsr()
        A.sort_indices()
        rows, indptr, col, val, asum, cnt = C.ref_rows(sub)
        assert np.array_equal(indptr, A.indptr) and np.array_equal(col, A.indices)
        assert np.all(np.abs(val - A.data) <= (cnt + 2) * 2.0**-53 * asum)
    A = C.spd_case()
    K = _assemble(A.groups, A.ndof)[A.loc_dof_eff][:, A.loc_dof_eff].toarray()
    assert np.linalg.eigvalsh(K).min() > 0
