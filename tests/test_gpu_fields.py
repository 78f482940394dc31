"""Field recovery on the device (csrc/fields.cuh, HexFields) against its host restatement (tests/fields_cases.py): element
strain and stress bit for bit on every brick edge (sizes one element before, on and after a brick edge per axis, with and
without the clamped face, uniform and field), principal values to the accuracy of acos, every output subset the same
bits as the full pass, nodal sums bit for bit against np.bincount of the GPU's own element values with exact counts, an
MG-PCG solve of a voxel box followed by the recovery, and refusals."""
import ctypes

import numpy as np
import pytest

from tests import fields_cases as C

pytestmark = pytest.mark.gpu

# bricks of 32 x 4 x 2 elements (kFdBX/BY/BZ)
BOXES = [
    ((1, 1, 1), (0, 0, 0), (1, 1, 1)),
    ((3, 2, 2), (2, 1, 1), (1, 1, 1)),
    ((31, 3, 1), (0, 0, 0), (31, 3, 1)),
    ((32, 4, 2), (0, 0, 0), (32, 4, 2)),
    ((33, 5, 3), (0, 0, 0), (33, 5, 3)),
    ((40, 9, 9), (7, 2, 3), (31, 5, 2)),
    ((40, 9, 9), (8, 1, 1), (32, 3, 3)),
    ((70, 9, 9), (3, 0, 0), (65, 9, 5)),
]
MATERIALS = [dict(h=1.0, E=1.0, nu=0.3), dict(h=0.37, E=2.5, nu=0.45)]
ALL = ("strain", "stress", "ps", "pe")


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def _block(box, mat):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    return HexBlock(*box, **mat)


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _check_principal(P, s):
    """P within 1e-7 max|s| of the restatement per element, ordered, P2 the clamped (I1 - P1) - P3 of the GPU's own values."""
    R = C.principal(s)
    scale = np.maximum(np.max(np.abs(s), axis=1), 1e-300)
    assert np.all(np.isfinite(P))
    assert np.max(np.max(np.abs(P - R), axis=1) / scale) <= 1e-7
    assert np.all(P[:, 0] >= P[:, 1]) and np.all(P[:, 1] >= P[:, 2])
    I1 = (s[:, 0] + s[:, 1]) + s[:, 2]
    assert _bits(P[:, 1], np.minimum(np.maximum((I1 - P[:, 0]) - P[:, 2], P[:, 2]), P[:, 0]))


@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("field", [False, True])
@pytest.mark.parametrize("mat", [0, 1])
def test_element_fields_bit_identical(cuda, box, field, mat):
    from pcg_mpi_solver_b200 import HexFields
    blk = _block(box, MATERIALS[mat])
    rng = np.random.default_rng(hash((box, field, mat)) % 2**32)
    f = rng.uniform(0.01, 100.0, tuple(reversed(blk.ne))) if field else None
    x = rng.standard_normal(blk.n) * 10.0 ** rng.integers(-3, 3, blk.n)
    out = {k: v.cpu().numpy() for k, v in HexFields(blk, device=cuda, E_field=f).element(_t(x, cuda)).items()}
    eps = C.strain(blk, x)
    sig = C.stress(blk, eps, f)
    assert _bits(out["strain"], eps) and _bits(out["stress"], sig)
    _check_principal(out["ps"], sig)
    _check_principal(out["pe"], eps)


@pytest.mark.parametrize("box", [BOXES[4], BOXES[7]])
def test_every_subset_gives_the_full_pass_bits(cuda, box):
    from pcg_mpi_solver_b200 import HexFields
    blk = _block(box, MATERIALS[1])
    rng = np.random.default_rng(5)
    F = HexFields(blk, device=cuda, E_field=rng.uniform(0.5, 20.0, tuple(reversed(blk.ne))))
    x = _t(rng.standard_normal(blk.n), cuda)
    full = {k: v.cpu().numpy() for k, v in F.element(x).items()}
    for m in range(1, 16):
        sub = tuple(k for i, k in enumerate(ALL) if (m >> i) & 1)
        got = F.element(x, sub)
        assert sorted(got) == sorted(sub)
        for k in sub:
            assert _bits(got[k].cpu().numpy(), full[k]), (sub, k)


def _nodal_raw(F, x, kind, cuda):
    """(work, out) of pcgb_fields_nodal through the C ABI, work = (sum_0, sum_1, sum_2, count) per node."""
    import torch
    from pcg_mpi_solver_b200 import _lib
    work = torch.full((F.n_nodes, 4), float("nan"), dtype=torch.float64, device=cuda)
    out = torch.full((F.n_nodes, 3), float("nan"), dtype=torch.float64, device=cuda)
    _lib.check(_lib.load().pcgb_fields_nodal(F._h, _lib.ptr(x), kind, None, _lib.ptr(work), _lib.ptr(out), _lib.stream_ptr()))
    return work.cpu().numpy(), out.cpu().numpy()


@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("field", [False, True])
def test_nodal_average_bit_identical(cuda, box, field):
    from pcg_mpi_solver_b200 import HexFields
    blk = _block(box, MATERIALS[0])
    rng = np.random.default_rng(17)
    f = rng.uniform(0.01, 100.0, tuple(reversed(blk.ne))) if field else None
    F = HexFields(blk, device=cuda, E_field=f)
    x = _t(rng.standard_normal(blk.n), cuda)
    el = F.element(x, ("ps", "pe"))
    nx, ny, nz = blk.ne
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    inc = lambda l, n: np.where((l == 0) | (l == n), 1, 2) if n > 1 else np.ones_like(l)   # noqa: E731
    count = (inc(lx, nx) * inc(ly, ny) * inc(lz, nz)).ravel().astype(float)
    for kind, name in ((0, "ps"), (1, "pe")):
        S = C.nodal_sums(blk, el[name].cpu().numpy())
        work, out = _nodal_raw(F, x, kind, cuda)
        assert _bits(work, S) and np.array_equal(work[:, 3], count)
        assert _bits(out, C.nodal_average(S))
        assert _bits(F.nodal(x, "stress" if kind == 0 else "strain").cpu().numpy(), out)


def test_solve_then_recover(cuda):
    """MG-PCG on the index-free operator of an inclusion_field box, then every field from its x."""
    from pcg_mpi_solver_b200 import HexFields
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, inclusion_field, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ng = (32, 16, 16)
    blk = HexBlock(ng, (0, 0, 0), ng, h=1.0 / ng[0])
    f = inclusion_field(ng, fraction=0.3, radii=(1.5, 4.0), E_inclusion=10.0, seed=2)
    op = SubdomainOperator(generate_box_operator(blk, device=cuda, E_field=f))
    mg = HexMultigrid(op, blk, E_field=f)
    x, info = op.solve(load_vector(blk, device=cuda), mg, 1e-10, 200)
    assert info.flag == 0
    F = HexFields(blk, device=cuda, E_field=f)
    out = {k: v.cpu().numpy() for k, v in F.element(x).items()}
    xh = x.cpu().numpy()
    eps = C.strain(blk, xh)
    sig = C.stress(blk, eps, f)
    assert _bits(out["strain"], eps) and _bits(out["stress"], sig)
    _check_principal(out["ps"], sig)
    _check_principal(out["pe"], eps)
    for kind, name in (("stress", "ps"), ("strain", "pe")):
        nod = F.nodal(x, kind).cpu().numpy()
        assert np.all(np.isfinite(nod))
        assert _bits(nod, C.nodal_average(C.nodal_sums(blk, out[name])))
    # the load pulls the free end down: the largest principal stress sits at the clamped face, in tension
    assert np.max(out["ps"][:, 0]) > 0 > np.min(out["ps"][:, 2])


def test_refusals(cuda):
    import torch
    from pcg_mpi_solver_b200 import HexFields, _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    from pcg_mpi_solver_b200.solver import Communicator, make_halo
    blk = HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4))
    F = HexFields(blk, device=cuda)
    for bad in (torch.zeros(blk.n - 3, dtype=torch.float64, device=cuda), torch.zeros(blk.n, dtype=torch.float32, device=cuda),
                torch.zeros(blk.n, dtype=torch.float64)):
        with pytest.raises(ValueError):
            F.element(bad)
        with pytest.raises(ValueError):
            F.nodal(bad)
    with pytest.raises(ValueError):
        F.element(torch.zeros(blk.n, dtype=torch.float64, device=cuda), ("stress", "vonmises"))
    with pytest.raises(ValueError):
        F.nodal(torch.zeros(blk.n, dtype=torch.float64, device=cuda), "ps")
    for v in (0.0, -1.0, float("nan"), float("inf")):
        f = np.ones((4, 5, 6))
        f[2, 3, 1] = v
        with pytest.raises(_lib.PcgbError):
            HexFields(blk, device=cuda, E_field=f)
    with pytest.raises(ValueError):
        HexFields(blk, device=cuda, E_field=np.ones((4, 5, 5)))
    lib = _lib.load()
    h = ctypes.c_void_p()
    box = blk.cbox()
    for args in ((0.0, 1.0, 0.3), (1.0, -1.0, 0.3), (1.0, 1.0, 0.5), (float("nan"), 1.0, 0.3)):
        assert lib.pcgb_fields_create(ctypes.byref(box), *args, None, ctypes.byref(h)) == -1 and not h
    outside = HexBlock((6, 5, 4), (2, 0, 0), (6, 5, 4)).cbox()
    assert lib.pcgb_fields_create(ctypes.byref(outside), 1.0, 1.0, 0.3, None, ctypes.byref(h)) == -1 and not h
    # x overlapping an output, work overlapping out
    x = torch.zeros(blk.n + 6 * 120, dtype=torch.float64, device=cuda)
    assert lib.pcgb_fields_element(F._h, _lib.ptr(x), _lib.ptr(x) + 8 * blk.n - 8, None, None, None, _lib.stream_ptr()) == -1
    w = torch.zeros(4 * F.n_nodes + 3 * F.n_nodes, dtype=torch.float64, device=cuda)
    assert lib.pcgb_fields_nodal(F._h, _lib.ptr(x), 0, None, _lib.ptr(w), _lib.ptr(w) + 8, _lib.stream_ptr()) == -1
    assert lib.pcgb_fields_nodal(F._h, _lib.ptr(x), 2, None, _lib.ptr(w), _lib.ptr(w) + 32 * F.n_nodes, _lib.stream_ptr()) == -1
    # a halo plan over vectors that are not 4 per node
    comm = Communicator(0, 1, None, device=cuda)
    for n in (3 * F.n_nodes, 4 * F.n_nodes + 4):
        halo = make_halo(comm, [], [], n)
        try:
            assert lib.pcgb_fields_nodal(F._h, _lib.ptr(x), 0, halo, _lib.ptr(w), _lib.ptr(w) + 32 * F.n_nodes, _lib.stream_ptr()) == -1
            assert b"4 per node" in lib.pcgb_last_error()
        finally:
            lib.pcgb_halo_destroy(halo)
    halo = make_halo(comm, [], [], 4 * F.n_nodes)    # the right length is accepted (no neighbours: nothing to add)
    try:
        assert lib.pcgb_fields_nodal(F._h, _lib.ptr(x), 0, halo, _lib.ptr(w), _lib.ptr(w) + 32 * F.n_nodes, _lib.stream_ptr()) == 0
    finally:
        torch.cuda.synchronize()
        lib.pcgb_halo_destroy(halo)
