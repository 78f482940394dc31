"""The host restatement of periodic homogenisation (tests/homog_cases.py) against physics: the uniform cell, a laminate
against its closed form, symmetry, the Hill-Mandel energy identity, the Voigt-Reuss bounds, invariance under cyclic
shifts, a 90-degree rotation and the translation null space.  No GPU."""
import numpy as np
import pytest

from pcg_mpi_solver_b200.hexmesh import inclusion_field
from tests import homog_cases as H

NU = 0.3


def test_uniform_cell_is_the_material():
    ne, h, E = (3, 4, 2), 0.5, 2.5
    for j in range(6):
        b = H.load(ne, np.eye(6)[j], h, E, NU)
        assert np.abs(b).max() <= 1e-13 * E * h * h
    C = H.effective_stiffness(ne, h, E, NU)
    D = E * H.d_matrix(NU)
    assert np.abs(C - D).max() <= 1e-12 * np.abs(D).max()
    lam, mu = D[0, 1], D[3, 3]
    assert np.isclose(D[0, 0], lam + 2 * mu) and np.isclose(lam, E * NU / ((1 + NU) * (1 - 2 * NU)))


def laminate_field(ne, E_layers):
    nx, ny, nz = ne
    f = np.empty((nz, ny, nx))
    for z in range(nz):
        f[z] = E_layers[z % len(E_layers)]
    return f


def test_laminate_matches_closed_form():
    ne = (4, 3, 8)
    E_layers = [1.0, 1.0, 7.0, 3.0]
    C = H.effective_stiffness(ne, 0.25, 1.0, NU, laminate_field(ne, E_layers))
    ref = H.laminate(E_layers, [0.25] * 4, NU)
    assert np.abs(C - ref).max() <= 1e-10 * np.abs(ref).max()


@pytest.fixture(scope="module")
def inclusion_case():
    ne = (6, 5, 4)
    f = inclusion_field(ne, fraction=0.3, radii=(1.0, 2.0), E_inclusion=10.0, seed=3)
    C, us = H.effective_stiffness(ne, 1.0 / 6, 1.0, NU, f, return_u=True)
    return ne, f, C, us


def test_symmetric(inclusion_case):
    _, _, C, _ = inclusion_case
    assert np.abs(C - C.T).max() <= 1e-10 * np.abs(C).max()


def test_hill_mandel(inclusion_case):
    ne, f, C, us = inclusion_case
    for i in range(6):
        for j in range(6):
            w = H.energy(ne, us[i], np.eye(6)[i], us[j], np.eye(6)[j], 1.0 / 6, 1.0, NU, f)
            assert abs(w - C[i, j]) <= 1e-10 * np.abs(C).max(), (i, j, w, C[i, j])


def test_voigt_reuss_bounds(inclusion_case):
    _, f, C, _ = inclusion_case
    D = H.d_matrix(NU)
    Cs = 0.5 * (C + C.T)
    tol = 1e-10 * np.abs(C).max()
    assert np.linalg.eigvalsh(f.mean() * D - Cs).min() >= -tol
    assert np.linalg.eigvalsh(Cs - D / np.mean(1.0 / f)).min() >= -tol
    assert np.linalg.eigvalsh(f.mean() * D - Cs).max() > 1e-3      # strictly inside: the field is not uniform


def test_cyclic_shift_invariance(inclusion_case):
    ne, f, C, _ = inclusion_case
    for axis, k in ((2, 1), (1, 2), (0, 3)):
        Cr = H.effective_stiffness(ne, 1.0 / 6, 1.0, NU, np.roll(f, k, axis=axis))
        assert np.abs(Cr - C).max() <= 1e-10 * np.abs(C).max(), axis


def test_rotation_permutes(inclusion_case):
    ne, f, C, _ = inclusion_case
    # G[z, Y, X] = F[z, ny - 1 - X, Y]: the material turned by +90 degrees about z, (x, y) -> (-y, x)
    g = np.ascontiguousarray(f[:, ::-1, :].transpose(0, 2, 1))
    Cr = H.effective_stiffness((ne[1], ne[0], ne[2]), 1.0 / 6, 1.0, NU, g)
    Q = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    assert np.abs(Cr - H.rotate_voigt(C, Q)).max() <= 1e-10 * np.abs(C).max()


def test_translations_are_the_null_space():
    ne = (3, 2, 4)
    f = inclusion_field(ne, fraction=0.4, radii=(1.0, 1.5), E_inclusion=5.0, seed=1)
    K = H.assemble(ne, 0.5, 1.0, NU, f)
    for d in range(3):
        t = np.zeros(K.shape[0])
        t[d::3] = 1.0
        assert np.abs(K @ t).max() <= 1e-13 * abs(K).max()
    # the load lies in K's range: its entries sum to 0 per direction
    b = H.load(ne, [0.3, -0.2, 0.1, 0.5, -0.4, 0.2], 0.5, 1.0, NU, f)
    for d in range(3):
        assert abs(b[d::3].sum()) <= 1e-13 * np.abs(b).sum()


def test_average_restatement_is_the_mean():
    rng = np.random.default_rng(0)
    for ne in ((2, 2, 2), (33, 5, 3), (64, 8, 4)):
        v = rng.standard_normal((int(np.prod(ne)), 3))
        assert np.allclose(H.ref_average(ne, v), v.mean(axis=0), rtol=1e-12, atol=1e-14)
