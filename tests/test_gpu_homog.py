"""Periodic-cell homogenisation on the device (DESIGN §2.13): the periodic index-free operator entrywise against its
long-double restatement at the brick edges (NaN-filled outputs), its diagonal bit for bit, the macroscopic-strain load,
symmetry, PCG solves against scipy, the fused average bit for bit against its stated order, effective_stiffness against
the host restatement and physics, and refusals that leak nothing."""
import ctypes
import gc

import numpy as np
import pytest

from tests import homog_cases as H

pytestmark = pytest.mark.gpu

# nodes per axis = elements per axis; brick 32 x 4 x 2 nodes: one below, at and one above on each axis, and the minimal cell
CELLS = [(2, 2, 2), (31, 3, 2), (32, 4, 2), (33, 5, 3), (3, 7, 4), (65, 4, 5)]
MATERIALS = [dict(nu=0.2, E=1.0, h=1.0), dict(nu=0.45, E=2.5, h=0.37)]
STRAIN = np.array([0.3, -0.7, 1.1, 0.45, -0.25, 0.8])


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _nan(n, cuda):
    import torch
    return torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)


def _bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _setup(ne, field, mat, cuda, seed=0):
    from pcg_mpi_solver_b200.hexmesh import PeriodicCell, generate_periodic_operator
    cell = PeriodicCell(ne, **mat)
    f = np.random.default_rng(seed).uniform(0.01, 100.0, tuple(reversed(ne))) if field else None
    ck = H.ck_of(ne, cell.h, cell.E, f)
    return cell, f, ck, generate_periodic_operator(cell, device=cuda, E_field=f)


@pytest.mark.parametrize("ne", CELLS)
@pytest.mark.parametrize("field", [False, True])
@pytest.mark.parametrize("mat", [0, 1])
def test_operator_diagonal_and_load(ne, field, mat, cuda):
    cell, f, ck, op = _setup(ne, field, MATERIALS[mat], cuda, seed=mat)
    nu = cell.nu
    rng = np.random.default_rng(7)
    x = rng.standard_normal(cell.n) * 10.0 ** rng.integers(-50, 50, cell.n)
    x[rng.random(cell.n) < 0.1] = -0.0
    y = _nan(cell.n, cuda)
    op.apply_local(_t(x, cuda), out=y)
    rows = np.arange(cell.n)
    H.assert_rows(y.cpu().numpy(), H.ref_rows(ne, rows, H.x_fetch(ne, x), ck, nu))
    d = op.diagonal()
    assert _bits(d.cpu().numpy(), H.ref_diag(ne, ck, nu))
    b = _nan(cell.n, cuda)
    op.load(STRAIN, out=b)
    y, s, k = H.ref_rows(ne, rows, H.ubar_table(STRAIN, cell.h), ck, nu)
    H.assert_rows(b.cpu().numpy(), (-y, s, k))
    # the element-wise host load (absolute corner values per element) is the same vector up to rounding
    ref = H.load(ne, STRAIN, cell.h, cell.E, nu, f)
    assert np.abs(b.cpu().numpy() - ref).max() <= 1e-12 * np.abs(ck).max() * cell.h * np.abs(STRAIN).max() * 24
    assert op.spmv_bytes() == 16 * cell.n + (8 * cell.n_elements if field else 0)


@pytest.mark.parametrize("field", [False, True])
def test_symmetric(field, cuda):
    cell, _, _, op = _setup((9, 6, 5), field, MATERIALS[1], cuda)
    rng = np.random.default_rng(1)
    x, y = rng.standard_normal(cell.n), rng.standard_normal(cell.n)
    kx, ky = op.apply_local(_t(x, cuda)).cpu().numpy(), op.apply_local(_t(y, cuda)).cpu().numpy()
    assert abs(y @ kx - x @ ky) <= 1e-13 * np.abs(y).sum() * np.abs(kx).max() + 1e-13 * abs(y @ kx)
    for dd in range(3):                                 # the translations are the null space
        t = np.zeros(cell.n)
        t[dd::3] = 1.0
        assert np.abs(op.apply_local(_t(t, cuda)).cpu().numpy()).max() <= 1e-12 * np.abs(kx).max() / np.abs(x).max()


@pytest.mark.parametrize("ne", [(4, 3, 5), (6, 6, 6)])
def test_solves_match_scipy(ne, cuda):
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    from pcg_mpi_solver_b200.hexmesh import inclusion_field
    cell, _, _, _ = _setup(ne, False, MATERIALS[0], cuda)
    f = inclusion_field(ne, fraction=0.3, radii=(1.0, 2.0), E_inclusion=10.0, seed=2)
    from pcg_mpi_solver_b200.hexmesh import generate_periodic_operator
    op = generate_periodic_operator(cell, device=cuda, E_field=f)
    sop = SubdomainOperator(op)
    minv = sop.jacobi()
    K = H.assemble(ne, cell.h, cell.E, cell.nu, f)
    for j in (0, 3):
        strain = np.eye(6)[j]
        x, info = sop.solve(op.load(strain), minv, 1e-11, 5000)
        assert info.flag == 0
        ref = H.solve(K, H.load(ne, strain, cell.h, cell.E, cell.nu, f))
        xg = x.cpu().numpy()
        for dd in range(3):                             # remove the mean translation of both
            xg[dd::3] -= xg[dd::3].mean()
            ref[dd::3] -= ref[dd::3].mean()
        assert np.abs(xg - ref).max() <= 1e-8 * np.abs(ref).max()


@pytest.mark.parametrize("ne", [(2, 2, 2), (33, 5, 3), (64, 8, 4), (40, 41, 9)])
@pytest.mark.parametrize("field", [False, True])
def test_average_bits(ne, field, cuda):
    from pcg_mpi_solver_b200.fields import PeriodicFields
    cell, f, _, _ = _setup(ne, field, MATERIALS[1], cuda, seed=3)
    F = PeriodicFields(cell, device=cuda, E_field=f)
    x = _t(np.random.default_rng(4).standard_normal(cell.n), cuda)
    el = F.element(x, STRAIN, fields=("strain", "stress"))
    es, ss = F.average(x, STRAIN)
    vals = np.concatenate([el["strain"].cpu().numpy(), el["stress"].cpu().numpy()], axis=1)
    ref = H.ref_average(ne, vals)
    assert _bits(es, ref[:6]) and _bits(ss, ref[6:])
    es2, ss2 = F.average(x, STRAIN)
    assert _bits(es, es2) and _bits(ss, ss2)
    # the element fields are the host restatement's (the explicit operation order of fields.cuh) to rounding
    hs, hsg = H.element_fields(ne, x.cpu().numpy(), STRAIN, cell.h, cell.E, cell.nu, f)
    assert np.allclose(vals[:, :6], hs, rtol=1e-12, atol=1e-12 * np.abs(hs).max())
    assert np.allclose(vals[:, 6:], hsg, rtol=1e-12, atol=1e-12 * np.abs(hsg).max())
    # the fluctuation averages out: <strain> = eps_bar (tensor shears) to rounding
    assert np.allclose(es, np.concatenate([STRAIN[:3], 0.5 * STRAIN[3:]]), atol=1e-12 * np.abs(hs).max())


def test_effective_stiffness_uniform_and_laminate(cuda):
    from pcg_mpi_solver_b200 import effective_stiffness
    from pcg_mpi_solver_b200.hexmesh import PeriodicCell
    cell = PeriodicCell((5, 4, 3), h=0.5, E=2.5, nu=0.3)
    C, infos = effective_stiffness(cell, device=cuda)
    assert all(i.flag == 0 and i.iters == 0 for i in infos)
    assert np.abs(C - cell.E * H.d_matrix(cell.nu)).max() <= 1e-14 * cell.E
    ne = (4, 3, 8)
    E_layers = [1.0, 1.0, 7.0, 3.0]
    f = np.empty(tuple(reversed(ne)))
    for z in range(ne[2]):
        f[z] = E_layers[z % 4]
    lam = PeriodicCell(ne, h=0.25, nu=0.3)
    C, infos = effective_stiffness(lam, E_field=f, tol=1e-10, device=cuda)
    ref = H.effective_stiffness(ne, 0.25, 1.0, 0.3, f)
    assert all(i.flag == 0 for i in infos)
    assert np.abs(C - ref).max() <= 1e-7 * np.abs(ref).max()
    assert np.abs(C - H.laminate(E_layers, [0.25] * 4, 0.3)).max() <= 1e-7 * np.abs(ref).max()
    assert np.abs(C - C.T).max() <= 1e-7 * np.abs(C).max()


def test_effective_stiffness_inclusion_64(cuda):
    from pcg_mpi_solver_b200 import effective_stiffness
    from pcg_mpi_solver_b200.hexmesh import PeriodicCell, inclusion_field
    ne = (64, 64, 64)
    cell = PeriodicCell(ne, h=1.0 / 64, nu=0.2)
    f = inclusion_field(ne, E_inclusion=10.0)
    C, infos, fields = effective_stiffness(cell, E_field=f, device=cuda, return_fields=True)
    assert [i.flag for i in infos] == [0] * 6, [(i.flag, i.iters, i.relres) for i in infos]
    assert all(i.iters > 0 for i in infos)
    D = H.d_matrix(cell.nu)
    Cs = 0.5 * (C + C.T)
    assert np.abs(C - C.T).max() <= 1e-6 * np.abs(C).max()
    assert np.linalg.eigvalsh(f.mean() * D - Cs).min() >= -1e-7 * np.abs(C).max()
    assert np.linalg.eigvalsh(Cs - D / np.mean(1.0 / f)).min() >= -1e-7 * np.abs(C).max()
    S = fields["strain"]
    assert np.abs(S - np.diag([1, 1, 1, 0.5, 0.5, 0.5])).max() <= 1e-10
    print("C_eff 64^3 contrast 10:", np.array2string(C, precision=5), "iterations", [i.iters for i in infos])


def test_refusals_leak_nothing(cuda):
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.fields import PeriodicFields
    from pcg_mpi_solver_b200.hexmesh import PeriodicCell, generate_periodic_operator, hex_element_stiffness
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    lib = _lib.load()
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(cuda)
    free0, _ = torch.cuda.mem_get_info(cuda)
    for ne in ((1, 4, 4), (4, 1, 4), (4, 4, 1), (0, 4, 4)):
        with pytest.raises(_lib.PcgbError):
            generate_periodic_operator(PeriodicCell(ne), device=cuda)
        with pytest.raises(_lib.PcgbError):
            PeriodicFields(PeriodicCell(ne), device=cuda)
    cell = PeriodicCell((5, 4, 3), h=0.5)
    ke = np.ascontiguousarray(hex_element_stiffness())
    kep = ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    h = ctypes.c_void_p()
    for ng, e0, ne in (((6, 4, 3), (0, 0, 0), (5, 4, 3)), ((5, 4, 3), (1, 0, 0), (5, 4, 3))):
        box = _lib.HexBox()
        for a in range(3):
            box.ng[a], box.e0[a], box.ne[a] = ng[a], e0[a], ne[a]
        assert lib.pcgb_hexop_create_periodic(ctypes.byref(box), kep, 1.0, None, ctypes.byref(h)) == -1 and not h
        assert lib.pcgb_fields_create_periodic(ctypes.byref(box), 1.0, 1.0, 0.3, None, ctypes.byref(h)) == -1 and not h
    for v in (0.0, -1.0, float("nan"), float("inf")):
        f = np.ones((3, 4, 5))
        f[2, 3, 4] = v
        with pytest.raises(_lib.PcgbError):
            generate_periodic_operator(cell, device=cuda, E_field=f)
        with pytest.raises(_lib.PcgbError):
            PeriodicFields(cell, device=cuda, E_field=f)
    with pytest.raises(ValueError):
        generate_periodic_operator(cell, device=cuda, E_field=np.ones((3, 4, 4)))
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(cuda) == before
    assert torch.cuda.mem_get_info(cuda)[0] >= free0
    op = generate_periodic_operator(cell, device=cuda)
    F = PeriodicFields(cell, device=cuda)
    x = torch.zeros(cell.n, dtype=torch.float64, device=cuda)
    for bad in (torch.zeros(cell.n + 3, dtype=torch.float64, device=cuda), torch.zeros(cell.n, dtype=torch.float64),
                torch.zeros(cell.n, dtype=torch.float32, device=cuda)):
        with pytest.raises(ValueError):
            F.average(bad, STRAIN)
        with pytest.raises(ValueError):
            F.element(bad, STRAIN)
    with pytest.raises(ValueError):
        F.average(x, STRAIN[:5])
    with pytest.raises(ValueError):
        F.nodal(x)
    sop = SubdomainOperator(op)
    with pytest.raises(ValueError, match="periodic"):
        HexMultigrid(sop, cell)
    # the box's handles and the periodic ones do not mix
    from pcg_mpi_solver_b200.fields import HexFields
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator
    blk = HexBlock((5, 4, 3), (0, 0, 0), (5, 4, 3))
    hb = generate_box_operator(blk, device=cuda)
    dp = ctypes.POINTER(ctypes.c_double)
    e = np.ascontiguousarray(STRAIN)
    out = np.zeros(6)
    assert lib.pcgb_hexop_periodic_load(hb.handle, e.ctypes.data_as(dp), 1.0, _lib.ptr(x), None) == -1
    assert lib.pcgb_hexop_periodic_load(op.handle, e.ctypes.data_as(dp), 0.0, _lib.ptr(x), None) == -1
    assert lib.pcgb_fields_average(HexFields(blk, device=cuda)._h, _lib.ptr(x), e.ctypes.data_as(dp), out.ctypes.data_as(dp),
                                   out.ctypes.data_as(dp), None) == -1
    assert lib.pcgb_fields_element(F._h, _lib.ptr(x), _lib.ptr(x), None, None, None, None) == -1
    assert lib.pcgb_fields_nodal(F._h, _lib.ptr(x), 0, None, _lib.ptr(x), _lib.ptr(x), None) == -1
    for bad in (torch.zeros(cell.n + 1, dtype=torch.float64, device=cuda), torch.zeros(cell.n, dtype=torch.float64),
                torch.zeros(2 * cell.n, dtype=torch.float64, device=cuda)[::2]):
        with pytest.raises(ValueError):
            op.load(STRAIN, out=bad)
    # the C ABI refuses a multigrid on a periodic solver even when the row counts agree (8x5x5 cell, 8x4x4 box: 600)
    per = generate_periodic_operator(PeriodicCell((8, 5, 5)), device=cuda)
    psop = SubdomainOperator(per)
    b8 = HexBlock((8, 4, 4), (0, 0, 0), (8, 4, 4)).cbox()
    assert 3 * 8 * 5 * 5 == HexBlock((8, 4, 4), (0, 0, 0), (8, 4, 4)).n
    mg = ctypes.c_void_p()
    minv = psop.jacobi()
    assert lib.pcgb_mg_create(psop._solver, ctypes.byref(b8), kep, 1.0, 1.0, _lib.ptr(minv), 2, 0.25, ctypes.byref(mg)) == -1
    assert not mg and "periodic" in lib.pcgb_last_error().decode()
    with pytest.raises(_lib.PcgbError):                 # x overlaps an output
        _lib.check(lib.pcgb_fields_element_periodic(F._h, _lib.ptr(x), e.ctypes.data_as(dp), _lib.ptr(x), None, None, None, None),
                   "pcgb_fields_element_periodic")
