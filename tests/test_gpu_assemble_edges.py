"""The device CSR assembly (csrc/assemble.cuh) entrywise at its kernel edges.

The cases come from tests/asm_cases.py: pattern sizes 1..255 with and without signs, clamped dofs and Ck over four decades;
rows of exactly 2047 / 2048 candidate columns and a refused 2049; every bitonic size and distinct-column counts on both
sides of each multiple of 32; empty rows, clamped-only rows, empty groups, n = 0, a 200-element hub; group indices >= 256,
element indices >= 2^24, local index 255; scans over 1023 .. 3 * 2^20 + 17 rows; summation-order rows; elements that list
a dof twice; and a band matrix with more than 2^31 non-zeros.  Each is compared with C.ref_rows, a long-double restatement
of sum_e P_e^T (Ck_e S_e Ke S_e) P_e: row offsets and columns exactly, every value within (k + 2) 2^-53 sum |terms| (k
terms: a first-order bound on fp64 rounding that cannot flake), and a second assembly bit for bit."""
import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import asm_cases as C

pytestmark = pytest.mark.gpu

U = 2.0**-53
X_RTOL, ITER_SLACK, TOL, MAXITER = 1e-10, 2, 1e-13, 3000     # as test_gpu_pcg / test_gpu_spmv_edges


def _device(sub, cuda):
    from pcg_mpi_solver_b200.partition import assemble_csr_device
    return assemble_csr_device(sub, cuda)


def _entries(rp, rows):
    """Positions in col / val of the entries of `rows` (ascending), and their row lengths."""
    lens = rp[rows + 1] - rp[rows]
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    return np.repeat(rp[rows] - starts, lens) + np.arange(lens.sum(), dtype=np.int64), lens


def _check(sub, cuda, rows=None, what=""):
    """Device assembly of `sub` against C.ref_rows on `rows` (all rows by default), then a second assembly bit for bit.
    Returns the host copies (rowptr int64, col, val)."""
    import torch
    rp_d, col_d, val_d = _device(sub, cuda)
    assert rp_d.dtype == torch.int32 and rp_d.numel() == sub.n + 1
    rp, col, val = rp_d.cpu().numpy().astype(np.int64), col_d.cpu().numpy(), val_d.cpu().numpy()
    rows_, indptr, rc, rv, asum, cnt = C.ref_rows(sub, rows)
    if rows is None:
        assert np.array_equal(rp, indptr), (what, "row offsets")
    assert rp[0] == 0 and rp[-1] == col.size == val.size
    idx, lens = _entries(rp, rows_)
    assert np.array_equal(lens, np.diff(indptr)), (what, "row lengths", np.nonzero(lens != np.diff(indptr))[0][:5])
    assert np.array_equal(col[idx], rc), (what, "columns")
    first = np.zeros(idx.size, bool)
    first[indptr[:-1][lens > 0]] = True
    assert np.all((np.diff(col[idx]) > 0) | first[1:]), (what, "columns not strictly ascending")
    err = np.abs(val[idx].astype(np.longdouble) - rv)
    bound = (cnt + 2) * U * asum
    bad = np.nonzero(err > bound)[0]
    assert bad.size == 0, (what, "values", bad[:5], err[bad[:5]], bound[bad[:5]])
    rp2, col2, val2 = _device(sub, cuda)
    assert torch.equal(rp2, rp_d) and torch.equal(col2, col_d) and torch.equal(val2, val_d), (what, "not bit-reproducible")
    return rp, col, val


# ------------------------------------------------------------------------------------------------ pattern sizes
@pytest.mark.parametrize("nd", C.PATTERN_SIZES)
def test_pattern_sizes(cuda, nd):
    for variant in C.PATTERN_VARIANTS:
        _check(C.pattern_case(nd, variant), cuda, what=(nd, variant))


# ------------------------------------------------------------------------------------------------ candidate limit
def test_candidate_limit(cuda):
    """2047 and 2048 candidates assemble; 2049 is refused with a PcgbError naming the limit, 20 times without leaking device
    memory, and a valid assembly still passes afterwards."""
    import torch
    from pcg_mpi_solver_b200._lib import PcgbError
    for total in (2047, 2048):
        _check(C.candidate_case(total), cuda, what=total)
    bad = C.candidate_case(2049)
    _device(C.candidate_case(2048), cuda)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(cuda)[0]
    for _ in range(20):
        with pytest.raises(PcgbError, match="more than 2048 candidate columns"):
            _device(bad, cuda)
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info(cuda)[0] - free0) <= 4 << 20
    _check(C.candidate_case(2048), cuda, what="after refusals")


# ------------------------------------------------------------------------------------------------ bitonic / compaction
def test_bitonic_and_compaction_sizes(cuda):
    _check(C.bitonic_case(), cuda, what="bitonic")


# ------------------------------------------------------------------------------------------------ structural edges
def test_structural_edges(cuda):
    sub = C.structure_case()
    rp, col, val = _check(sub, cuda, what="structure")
    pos = np.full(sub.ndof, -1)
    pos[sub.loc_dof_eff] = np.arange(sub.n)
    e = pos[sub.extra["empty"]]
    assert np.all(rp[e + 1] == rp[e])
    lone = pos[sub.extra["lonely"]]
    assert np.all(rp[lone + 1] - rp[lone] == 1) and np.array_equal(col[rp[lone]], lone)
    rp0, col0, val0 = _device(C.no_rows_case(), cuda)
    assert rp0.tolist() == [0] and col0.numel() == 0 and val0.numel() == 0


# ------------------------------------------------------------------------------------------------ key fields
def test_group_index_above_255(cuda):
    _check(C.many_groups_case(), cuda, what="300 groups")


def test_local_index_255(cuda):
    _check(C.wide_pattern_case(), cuda, what="nd 255")


def test_element_index_above_2_24(cuda):
    """nd = 1, 2^24 + 3 elements: the rows of the elements >= 2^24 (and of e - 2^24) plus 3000 random rows against the
    reference; every row's structure exactly (a row is its own diagonal when an element touches it)."""
    import torch
    sub = C.many_elements_case()
    (g,) = sub.groups
    tail = np.arange(2**24, C.BIG_NE)
    rows = np.concatenate([g.loc_dof[0, tail], g.loc_dof[0, tail - 2**24], [0, sub.n - 1],
                           np.random.default_rng(5).integers(0, sub.n, 3000)])
    rp, col, val = _check(sub, cuda, rows=rows, what="2^24 elements")
    touched = np.bincount(g.loc_dof[0], minlength=sub.n) > 0
    assert np.array_equal(np.diff(rp), touched.astype(np.int64)) and np.array_equal(col, np.nonzero(touched)[0])
    del rp, col, val
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ scan lengths
@pytest.mark.parametrize("n", C.SCAN_SIZES)
def test_scan_lengths(cuda, n):
    _check(C.scan_case(n), cuda, what=n)


# ------------------------------------------------------------------------------------------------ summation order
def test_fixed_summation_order(cuda):
    """Exact products: every value equals, bit for bit, the fp64 sum in the documented (group, element, local index) order;
    the diagonal of the order rows is 0 in that order and 1 in k_asm_fill's order."""
    sub = C.order_case()
    rp, col, val = _check(sub, cuda, what="order")
    doc = C.ordered_sums(sub, "documented")
    rows = np.repeat(np.arange(sub.n), np.diff(rp))
    want = np.array([doc[(r, c)] for r, c in zip(rows.tolist(), col.tolist())])
    assert np.array_equal(val.view(np.int64), want.view(np.int64)), np.nonzero(val != want)[0][:10]
    for r in sub.extra["rows"]:
        assert val[rp[r] + np.searchsorted(col[rp[r]:rp[r + 1]], r)] == 0.0


# ------------------------------------------------------------------------------------------------ repeated dofs
def test_element_listing_a_dof_twice(cuda):
    """An element that lists a free dof twice (one pass, two passes, three times) is summed like the host COO assembly
    (partition._assemble): the reference bound for the device, twice it against the host, and bit-reproducible."""
    from pcg_mpi_solver_b200.partition import _assemble
    sub = C.duplicate_case()
    rp, col, val = _check(sub, cuda, what="duplicates")
    A = _assemble(sub.groups, sub.ndof)[sub.loc_dof_eff][:, sub.loc_dof_eff].tocsr()
    A.sort_indices()
    _, _, _, rv, asum, cnt = C.ref_rows(sub)
    assert np.array_equal(rp, A.indptr) and np.array_equal(col, A.indices)
    assert np.all(np.abs(val - A.data) <= 2 * (cnt + 2) * U * asum)


# ------------------------------------------------------------------------------------------------ solver
def test_device_assembled_operator_solves(cuda):
    """to_operator() with A unset assembles on the device; PCG on it against ref_pcg on the host assembly."""
    from pcg_mpi_solver_b200 import solve
    from pcg_mpi_solver_b200.partition import _assemble
    sub = C.spd_case()
    assert sub.A is None
    A = _assemble(sub.groups, sub.ndof)[sub.loc_dof_eff][:, sub.loc_dof_eff].tocsr()
    A.sort_indices()
    b = A @ np.random.default_rng(43).standard_normal(sub.n)
    minv = 1.0 / A.diagonal()
    hist = []
    ref = R.ref_pcg([R.CsrPart(A, b)], [minv], TOL, MAXITER, resvec=hist)
    assert ref["Flag"] == 0 and ref["Iter"] > 12
    op = sub.to_operator(device=cuda)
    x, flag, relres, iters, info = solve(op, b, minv, TOL, MAXITER, check_every=1, use_graph=False, record_resvec=True,
                                         return_info=True)
    assert flag == ref["Flag"] and abs(iters - ref["Iter"]) <= ITER_SLACK, (flag, iters, ref["Iter"])
    np.testing.assert_allclose(info.resvec[:12], np.array(hist)[:12], rtol=1e-9)
    assert np.linalg.norm(x - ref["X"][0]) <= X_RTOL * np.linalg.norm(ref["X"][0])


# ------------------------------------------------------------------------------------------------ offsets above 2^31
def test_int64_row_offsets(cuda):
    """band_case(INT64_NE): 5.6e6 rows, more than 2^31 non-zeros (26 GB of col + val).  rowptr stays int64 and equals the
    scan of the analytic row lengths; the row whose offsets contain 2^31, its neighbours, the first and last rows and 2000
    random rows match the reference entrywise."""
    import torch
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 40e9:
        pytest.skip("needs ~40 GB of free device memory")
    sub = C.band_case(C.INT64_NE)
    rp_d, col_d, val_d = _device(sub, cuda)
    lens = C.band_row_lengths(C.INT64_NE)
    assert rp_d.dtype == torch.int64 and int(rp_d[-1]) == lens.sum() >= 2**31
    rp = rp_d.cpu().numpy()
    assert np.array_equal(rp, np.concatenate([[0], np.cumsum(lens)]))
    r31 = int(np.searchsorted(rp, 2**31, side="right")) - 1
    assert rp[r31] <= 2**31 < rp[r31 + 1]
    rows = np.unique(np.concatenate([np.arange(r31 - 2, r31 + 3), [0, 1, sub.n - 2, sub.n - 1],
                                     np.random.default_rng(47).integers(0, sub.n, 2000)]))
    rows_, indptr, rc, rv, asum, cnt = C.ref_rows(sub, rows)
    idx_h, lens_h = _entries(rp, rows_)
    idx = torch.from_numpy(idx_h).to(cuda)
    col, val = col_d[idx].cpu().numpy(), val_d[idx].cpu().numpy()
    assert np.array_equal(lens_h, np.diff(indptr)) and np.array_equal(col, rc)
    assert np.all(np.abs(val.astype(np.longdouble) - rv) <= (cnt + 2) * U * asum)
    del rp_d, col_d, val_d, idx
    torch.cuda.empty_cache()
