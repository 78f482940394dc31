"""The index-free hex-box operator (csrc/hexop.cuh, HexBoxOperator) on the device: products and diagonals bit-identical to
the ordered EBE operator on every box edge (brick size +-1, odd and even nxf, uniform and field, two materials, signed zeros
and many decades), entrywise against the long-double restatement (tests/hexop_cases.py), Ke owned by the handle,
refusals that leak nothing, a sampled 512^3 box, PCG and MG-PCG bit-identical to the same solves on the ordered operator,
the oracle, launch counts and the committed 128^3 residual history."""
import gc
import json
import os

import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import hexop_cases as C

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# brick size 32 x 4 x 2 nodes (kHxBX/BY/BZ): nxf, ny + 1, nz + 1 one below, at and one above a multiple of it
BRICK_BOXES = [
    ((32, 3, 1), (0, 0, 0), (32, 3, 1)),      # nxf 32 (clamped face): even
    ((31, 3, 1), (0, 0, 0), (31, 3, 1)),      # nxf 31: odd
    ((33, 4, 2), (0, 0, 0), (33, 4, 2)),      # nxf 33: odd
    ((40, 9, 9), (8, 2, 3), (30, 2, 3)),      # nxf 31 (no clamped face)
    ((40, 9, 9), (8, 2, 3), (31, 4, 2)),      # nxf 32
    ((40, 9, 9), (7, 1, 1), (32, 7, 5)),      # nxf 33
    ((65, 8, 5), (0, 0, 0), (65, 8, 5)),
]
MATERIALS = [dict(nu=0.2, E=1.0, h=1.0), dict(nu=0.45, E=2.5, h=0.37)]


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _apply(E, x, cuda):
    """E applied to x into a NaN-filled output (every entry must be written)."""
    import torch
    y = torch.full((E.shape[0],), float("nan"), dtype=torch.float64, device=cuda)
    E.apply_local(_t(x, cuda), out=y)
    return y.cpu().numpy()


def _field(blk, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.01, 100.0, tuple(reversed(blk.ne)))


def _pair(blk, cuda, field):
    from pcg_mpi_solver_b200.hexmesh import generate_box_operator, generate_ebe
    return generate_box_operator(blk, device=cuda, E_field=field), generate_ebe(blk, device=cuda, ordered=True, E_field=field)


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


@pytest.mark.parametrize("box", C.BOXES + BRICK_BOXES)
@pytest.mark.parametrize("field", [False, True])
@pytest.mark.parametrize("mat", [0, 1])
def test_bit_identical_to_ordered(cuda, box, field, mat):
    """apply_local and diagonal() bit for bit (signed zeros included) against generate_ebe(ordered=True), and entrywise
    against the long-double restatement, for x with signed zeros over many decades and for a plain x."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    blk = HexBlock(*box, **MATERIALS[mat])
    f = _field(blk, sum(box[2]) + mat) if field else None
    H, O = _pair(blk, cuda, f)
    ck = (f.reshape(-1) * blk.h) if field else np.full(int(np.prod(blk.ne)), blk.E * blk.h)
    rng = np.random.default_rng(17 + mat)
    for x in (C.hard_x(blk.n, rng), rng.standard_normal(blk.n)):
        yh, yo = _apply(H, x, cuda), _apply(O, x, cuda)
        assert _bits(yh, yo)
        C.assert_rows(yh, blk, np.arange(blk.n), lambda i: x[i], lambda e: ck[e])
    assert _bits(H.diagonal().cpu().numpy(), O.diagonal().cpu().numpy())
    assert H.spmv_bytes() == 16 * blk.n + (8 * ck.size if field else 0)


def test_negative_zero_rows(cuda):
    """x = -0.0 everywhere: every product term is -0.0 or +0.0 as in the ordered kernel; y bit-equal (all +0.0)."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    blk = HexBlock((5, 4, 3), (0, 0, 0), (5, 4, 3), h=0.5)
    H, O = _pair(blk, cuda, None)
    x = np.full(blk.n, -0.0)
    assert _bits(_apply(H, x, cuda), _apply(O, x, cuda))


def test_ke_owned_by_the_handle(cuda):
    """Two live operators of different nu and E keep their products while generate_matrix, a Galerkin multigrid set-up and
    ordered EBE operators of other materials are built in between."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    b1 = HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4), h=0.25, E=1.0, nu=0.2)
    b2 = HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4), h=0.25, E=7.0, nu=0.45)
    H1, H2 = generate_box_operator(b1, device=cuda), generate_box_operator(b2, device=cuda)
    x = np.random.default_rng(3).standard_normal(b1.n)
    y1, y2 = _apply(H1, x, cuda), _apply(H2, x, cuda)
    assert not _bits(y1, y2)
    b3 = HexBlock((8, 8, 8), (0, 0, 0), (8, 8, 8), h=0.125, nu=0.33)
    A3 = generate_matrix(b3, device=cuda)
    op3 = SubdomainOperator(generate_matrix(b3, device=cuda))
    mg3 = HexMultigrid(op3, b3, E_field=np.full((8, 8, 8), 3.0))
    others = [generate_ebe(HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4), nu=nu), device=cuda, ordered=True) for nu in (0.1, 0.25, 0.4)]
    torch.cuda.synchronize()
    assert _bits(_apply(H1, x, cuda), y1) and _bits(_apply(H2, x, cuda), y2)
    _, O1 = _pair(b1, cuda, None)
    _, O2 = _pair(b2, cuda, None)
    assert _bits(y1, _apply(O1, x, cuda)) and _bits(y2, _apply(O2, x, cuda))
    del A3, op3, mg3, others


def test_refusals_leak_nothing(cuda):
    import ctypes
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, hex_element_stiffness
    blk = HexBlock((5, 4, 3), (0, 0, 0), (5, 4, 3), h=0.5)
    lib = _lib.load()
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(cuda)
    free0, _ = torch.cuda.mem_get_info(cuda)
    for bad in (np.ones((3, 4, 4)), np.ones((3, 4, 5), dtype=np.float32), torch.ones((3, 4, 5), dtype=torch.float64, device="meta"),
                [[1.0]]):
        with pytest.raises(ValueError):
            generate_box_operator(blk, device=cuda, E_field=bad)
    for v in (0.0, -1.0, float("nan"), float("inf")):
        f = np.ones((3, 4, 5))
        f[2, 3, 4] = v
        with pytest.raises(_lib.PcgbError):
            generate_box_operator(blk, device=cuda, E_field=f)
        with pytest.raises(_lib.PcgbError):
            generate_box_operator(blk, device=cuda, E_field=torch.from_numpy(f).to(cuda))
    ke = np.ascontiguousarray(hex_element_stiffness())
    kep = ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    h = ctypes.c_void_p()
    for ng, e0, ne in (((5, 4, 3), (0, 0, 0), (0, 4, 3)), ((5, 4, 3), (0, 0, 0), (5, 4, -1)), ((5, 4, 3), (1, 0, 0), (5, 4, 3)),
                       ((5, 4, 3), (-1, 0, 0), (2, 4, 3)), ((5, 4, 3), (0, 0, 2), (5, 4, 2))):
        box = HexBlock(ng, e0, ne).cbox()
        assert lib.pcgb_hexop_create(ctypes.byref(box), kep, 1.0, None, ctypes.byref(h)) == -1 and not h
    box = blk.cbox()
    for ck in (0.0, -2.0, float("nan"), float("inf")):
        assert lib.pcgb_hexop_create(ctypes.byref(box), kep, ck, None, ctypes.byref(h)) == -1 and not h
    assert lib.pcgb_hexop_create(None, kep, 1.0, None, ctypes.byref(h)) == -1
    assert lib.pcgb_solver_create_hexop(None, None, None, ctypes.byref(h)) == -1
    assert lib.pcgb_hexop_apply(None, None, None, None) == -1
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(cuda) == before
    assert torch.cuda.mem_get_info(cuda)[0] >= free0
    H = generate_box_operator(blk, device=cuda)
    buf = torch.zeros(2 * blk.n, dtype=torch.float64, device=cuda)
    for xo, yo in ((0, 0), (0, blk.n - 1), (blk.n - 1, 0), (1, 0)):
        with pytest.raises(_lib.PcgbError):
            H.apply_local(buf[xo:xo + blk.n], out=buf[yo:yo + blk.n])
    H.apply_local(buf[:blk.n], out=buf[blk.n:])           # adjacent, not overlapping


def test_large_box_sampled_rows_and_pcg(cuda):
    """512^3 (n = 404 227 584): a few thousand rows around the start, the middle, the end and on the clamped face against
    the long-double restatement, then 20 fixed Jacobi-PCG iterations."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    B = 512
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    need = 12 * 8 * blk.n + (2 << 30)
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB free device memory, {free / 2**30:.1f} GiB free")
    H = generate_box_operator(blk, device=cuda)
    g = torch.Generator(device=cuda).manual_seed(512)
    x = torch.randn(blk.n, dtype=torch.float64, device=cuda, generator=g)
    y = torch.full((blk.n,), float("nan"), dtype=torch.float64, device=cuda)
    H.apply_local(x, out=y)
    nxf = B
    face = 3 * ((np.arange(0, B + 1, 37)[:, None] * (B + 1) + np.arange(0, B + 1, 41)[None, :]).ravel() * nxf)
    rows = np.unique(np.concatenate([np.arange(3000), blk.n // 2 - 1500 + np.arange(3000), blk.n - 3000 + np.arange(3000),
                                     face, face + 1, face + 2]))
    yr = y[torch.from_numpy(rows).to(cuda)].cpu().numpy()
    C.assert_rows(yr, blk, rows, lambda i: x[torch.from_numpy(np.asarray(i)).to(cuda)].cpu().numpy(), lambda e: np.full(len(e), blk.h))
    del y
    op = SubdomainOperator(H)
    b = load_vector(blk, device=cuda)
    xs, info = op.solve(b, op.jacobi(), 0.0, 20, fixed_iters=True, record_resvec=True, check_every=10)
    assert info.loop_iters == 20 and np.isfinite(info.resvec).all() and info.resvec[0] == info.normb    # x0 = 0: r0 = b


def _solve_pair(blk, cuda, field, use_graph=True, check_every=8, tol=1e-10, maxiter=3000):
    """(x, info) of the same Jacobi-PCG on the new operator and on the ordered one."""
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    out = []
    for A in _pair(blk, cuda, field):
        op = SubdomainOperator(A)
        b = load_vector(blk, device=cuda)
        out.append(op.solve(b, op.jacobi(), tol, maxiter, record_resvec=True, trace=True, check_every=check_every, use_graph=use_graph))
    return out


def _same_solve(a, b):
    import torch
    (xa, ia), (xb, ib) = a, b
    assert torch.equal(xa, xb)
    assert _bits(ia.resvec, ib.resvec) and ia.iters == ib.iters and ia.flag == ib.flag and ia.relres == ib.relres
    assert ia.trace_total == ib.trace_total and ia.trace.tobytes() == ib.trace.tobytes()


@pytest.mark.parametrize("field", [False, True])
def test_pcg_bit_identical_to_ordered(cuda, field):
    """x, resvec and trace identical to the ordered operator's solve, for graph on/off x check_every 1/7; all four runs
    identical to each other."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    blk = HexBlock((20, 9, 7), (0, 0, 0), (20, 9, 7), h=1.0 / 20)
    f = _field(blk, 5) if field else None
    first = None
    for use_graph in (True, False):
        for ce in (1, 7):
            a, b = _solve_pair(blk, cuda, f, use_graph=use_graph, check_every=ce)
            assert a[1].flag == 0
            _same_solve(a, b)
            if first is None:
                first = a
            else:
                import torch
                assert torch.equal(a[0], first[0]) and _bits(a[1].resvec, first[1].resvec)


def test_pcg_matches_oracle_and_launches(cuda):
    import torch
    from pcg_mpi_solver_b200 import solve
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, generate_ebe, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock((9, 7, 5), (0, 0, 0), (9, 7, 5), h=1.0 / 9, nu=0.35, E=2.0)
    A = R.hex_box_csr(blk.ng, blk.e0, blk.ne, E=blk.E, nu=blk.nu, h=blk.h)
    op = SubdomainOperator(generate_box_operator(blk, device=cuda))
    b = load_vector(blk, device="cpu").numpy()
    resvec = []
    ref = R.ref_pcg([R.CsrPart(A, b)], [1.0 / A.diagonal()], 1e-12, 5000, resvec=resvec)
    x, flag, relres, iters, info = solve(op, b, "jacobi", 1e-12, 5000, return_info=True, record_resvec=True)
    assert flag == ref["Flag"] == 0 and abs(iters - ref["Iter"]) <= 2
    assert np.linalg.norm(x - ref["X"][0]) <= 1e-10 * np.linalg.norm(ref["X"][0])
    np.testing.assert_allclose(info.resvec[:12], np.asarray(resvec[:12]), rtol=1e-9)

    def per_iter(o):
        bd = load_vector(blk, device=cuda)
        ls = []
        for maxiter in (8, 16):
            _, inf = o.solve(bd, o.jacobi(), 1e-30, maxiter, fixed_iters=True, check_every=8)
            ls.append(inf.launches)
        return ls[1] - ls[0]

    po = per_iter(SubdomainOperator(generate_ebe(blk, device=cuda, ordered=True)))
    ph = per_iter(op)
    assert ph == po - 8, (ph, po)         # the ordered operator launches twice per application, this one once
    torch.cuda.synchronize()


def test_residual_history_128_matches_golden(cuda):
    """The bench's 128^3 box against the oracle's committed residual history, bit-identical to the ordered operator."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, generate_ebe, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 8 * 2**30:
        pytest.skip("needs 8 GiB free device memory")
    B = 128
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    b = load_vector(blk, device=cuda)
    gold = json.load(open(os.path.join(HERE, "golden", f"hex{B}_N1_resvec.json")))
    ref = np.array(gold["resvec"])
    runs = []
    for A in (generate_box_operator(blk, device=cuda), None):
        if A is None:
            gc.collect()
            A = generate_ebe(blk, device=cuda, ordered=True)
        op = SubdomainOperator(A)
        x, info = op.solve(b, op.jacobi(), 0.0, 40, fixed_iters=True, record_resvec=True, check_every=20)
        runs.append((x, info))
        del op, A
    np.testing.assert_allclose(runs[0][1].resvec[:11], ref[:11], rtol=1e-9)
    np.testing.assert_allclose(runs[0][1].resvec[:41], ref[:41], rtol=1e-7)
    assert torch.equal(runs[0][0], runs[1][0]) and _bits(runs[0][1].resvec, runs[1][1].resvec)


def _mg_pair(blk, cuda, field, coarsening):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    out = []
    for A in _pair(blk, cuda, field):
        op = SubdomainOperator(A)
        out.append((op, HexMultigrid(op, blk, E_field=field, coarsening=coarsening)))
    return out


@pytest.mark.parametrize("kind", ["default", "field", "any"])
def test_multigrid_bit_identical_to_ordered_fine_operator(cuda, kind):
    """lambda, one V-cycle and MG-PCG (x, resvec, trace) on the new fine operator equal the same HexMultigrid on the ordered
    operator bit for bit."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, load_vector
    ne = (15, 9, 7) if kind == "any" else (16, 8, 8)
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0])
    f = _field(blk, 21) if kind == "field" else None
    (oh, mh), (oo, mo) = _mg_pair(blk, cuda, f, "any" if kind == "any" else "even")
    assert mh.info()["lambda"] == mo.info()["lambda"]
    r = _t(np.random.default_rng(2).standard_normal(blk.n), cuda)
    assert torch.equal(mh.apply(r), mo.apply(r))
    b = load_vector(blk, device=cuda)
    _same_solve(oh.solve(b, mh, 1e-10, 500, record_resvec=True, trace=True), oo.solve(b, mo, 1e-10, 500, record_resvec=True, trace=True))
