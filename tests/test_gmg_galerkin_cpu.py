"""The host restatements of the two Galerkin hierarchies (voxel_cases.HostFieldMultigrid for E_field, gmg_any_cases.
HostAnyMultigrid for coarsening="any") at materials other than nu = 0.3: their level matrices against scipy P^T A P, the
three host V-cycles on one constant-field box, the scaling of the element matrices, and the indefinite coarsest matrix the
nu = 0.6 refusal rests on.  The device tests of tests/test_gpu_gmg_galerkin_edges.py depend on these."""
import numpy as np
import pytest

from tests import gmg_any_cases as A
from tests import gmg_cases as G
from tests import voxel_cases as V


def _ptap_field(f, h, nu):
    lv = G.levels_of(tuple(int(v) for v in reversed(f.shape)))
    mats = [V.field_csr(f, h, nu)]
    for l in range(len(lv) - 1):
        P = G.prolongation_matrix(lv[l])
        mats.append((P.T @ mats[-1] @ P).tocsr())
    return mats


@pytest.mark.parametrize("h", [0.125, 2.0])
@pytest.mark.parametrize("nu", [0.2, 0.45])
@pytest.mark.parametrize("path,ne", [("field", (16, 8, 12)), ("any", (25, 17, 9))])
def test_level_matrices_equal_ptap_at_other_materials(path, ne, nu, h):
    """Every level of a random field, the field path on an all-even box and the any rule on a box with odd and kept axes,
    against scipy P^T A P to 1e-13 of the row's largest entry."""
    f = V.random_field(ne, seed=sum(ne))
    got = V.level_matrices(f, h, nu) if path == "field" else A.level_matrices(f, h, nu)
    ref = _ptap_field(f, h, nu) if path == "field" else A.ptap_matrices(f, h, nu)
    assert len(got) == len(ref) >= 3
    for l, (M, Q) in enumerate(zip(got, ref)):
        diff = abs(M - Q).max(axis=1).toarray().ravel()
        rowmax = abs(Q).max(axis=1).toarray().ravel()
        assert np.all(diff <= 1e-13 * rowmax), (l, float(np.max(diff / rowmax)))


@pytest.mark.parametrize("nu", [0.2, 0.45])
def test_three_host_vcycles_agree_on_a_constant_field(nu):
    """A constant field c on 16^3, where the even and the any rule give the same levels (16x8x8 would not: the any rule
    goes on from 4x2x2 to 2x2x2), with the same lambda: HostFieldMultigrid and HostAnyMultigrid give the same V-cycle to
    1e-13, and both that of the rediscretised HostMultigrid(E = c) to 1e-12.  Rediscretised and Galerkin coarse matrices
    differ by rounding that grows down the levels (5.6e-15 of the largest entry on the coarsest at nu = 0.45), and the
    V-cycle carries it to 3.4e-13 there (3.1e-14 at nu = 0.2)."""
    ne, h, c = (16, 16, 16), 1.0 / 16, 7.5
    assert G.levels_of(ne) == A.levels(ne)
    f = A.uniform_field(ne, c)
    Hr = G.HostMultigrid(ne, h, E=c, nu=nu)
    Hf = V.HostFieldMultigrid(f, h, lambdas=Hr.lam, nu=nu)
    Ha = A.HostAnyMultigrid(f, h, lambdas=Hr.lam, nu=nu)
    u = np.random.default_rng(int(100 * nu)).standard_normal(Hr.A[0].n)
    ref, mf, ma = Hr.apply(u), Hf.apply(u), Ha.apply(u)
    assert np.linalg.norm(ma - mf) <= 1e-13 * np.linalg.norm(mf)
    for m in (mf, ma):
        assert np.linalg.norm(m - ref) <= 1e-12 * np.linalg.norm(ref), np.linalg.norm(m - ref) / np.linalg.norm(ref)


@pytest.mark.parametrize("path,ne", [("field", (16, 8, 12)), ("any", (25, 17, 9))])
def test_element_matrices_scale_exactly(path, ne):
    """The host Galerkin element matrices of 4 f are exactly 4 times those of f on every level (weights k/8, a power-of-two
    scale)."""
    f = V.random_field(ne, seed=1)
    fn = V.level_elements if path == "field" else A.level_elements
    for a, b in zip(fn(4.0 * f, 0.5, 0.45), fn(f, 0.5, 0.45)):
        assert np.array_equal(a, 4.0 * b)


@pytest.mark.parametrize("path,ne,uniform", [("field", A.BAD_NU_FIELD_BOX, False), ("any", A.BAD_NU_ANY_BOX, True),
                                             ("any", A.BAD_NU_ANY_BOX, False)])
def test_bad_nu_coarsest_matrix_is_indefinite(path, ne, uniform):
    """At nu = 0.6 the Galerkin coarsest matrix of each refusal box has a negative eigenvalue, so the device's coarse
    Cholesky factorisation must meet a non-positive pivot."""
    f = A.uniform_field(ne) if uniform else V.random_field(ne, seed=sum(ne))
    mats = V.level_matrices(f, 1.0 / ne[0], G.BAD_NU) if path == "field" else A.level_matrices(f, 1.0 / ne[0], G.BAD_NU)
    Ac = mats[-1].toarray()
    assert np.linalg.eigvalsh(0.5 * (Ac + Ac.T))[0] < 0
