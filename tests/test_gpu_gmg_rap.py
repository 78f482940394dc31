"""The rap multigrid hierarchy (HexMultigrid(coarse="rap"), pcgb_mg_create_field_rap, csrc/gmg_rap.cuh) against the CSR field
hierarchy of the same voxel model (HexMultigrid(E_field=f)): the fused level-1 product bit for bit against the three launches
it fuses and to rounding against the CSR level 1, level 1's D^-1 and every level >= 2 (CSR, D^-1, lambda) bit for bit, the
set-up's determinism, the V-cycle, MG-PCG, launch counts, device bytes, refusals, and MG-PCG on a 512^3 voxel model when
the GPU has the memory.

Largest errors seen are collected in STATS and printed by the last test (-rP)."""
import numpy as np
import pytest

from tests import voxel_cases as V

pytestmark = pytest.mark.gpu
STATS = {}


def _stat(key, v):
    STATS[key] = max(STATS.get(key, 0.0), float(v))


def _t(v, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _np(t):
    return t.cpu().numpy()


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def _field(ne, kind, contrast, seed=0):
    if kind == "inclusion":
        return V.two_phase(ne, contrast, seed=seed)
    f = V.random_field(ne, seed, 1.0, float(contrast)) if contrast > 1 else np.ones((ne[2], ne[1], ne[0]))
    return f


def _operator(blk, cuda, kind, field):
    from pcg_mpi_solver_b200.hexmesh import generate_box_operator, generate_ebe, generate_matrix
    if kind == "csr":
        return generate_matrix(blk, device=cuda, E_field=field)
    if kind == "hexop":
        return generate_box_operator(blk, device=cuda, E_field=field)
    return generate_ebe(blk, device=cuda, ordered=True, E_field=field)


def _setup(cuda, field, kind="hexop", degree=2, lo=0.25, both=True, minv=None):
    """(block, operator, rap hierarchy, CSR field hierarchy or None)"""
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = tuple(int(v) for v in reversed(field.shape))
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0])
    op = SubdomainOperator(_operator(blk, cuda, kind, field))
    mr = HexMultigrid(op, blk, degree=degree, lo=lo, E_field=field, coarse="rap", minv=minv)
    mc = HexMultigrid(op, blk, degree=degree, lo=lo, E_field=field, minv=minv) if both else None
    return blk, op, mr, mc


# level-1 widths around the 8 x 4 x 4 coarse-node brick: x over nx_1 = 6 / 8 / 10 free nodes, y and z over 5 / 7 / 9 nodes
BOXES = [(16, 16, 16), (16, 8, 12), (32, 32, 32), (64, 64, 64), (12, 8, 8), (20, 12, 16), (20, 16, 8)]
FIELDS = [("inclusion", 10), ("inclusion", 1000), ("random", 1), ("random", 10), ("random", 100), ("random", 1000)]


@pytest.mark.parametrize("ne", BOXES)
@pytest.mark.parametrize("fkind,contrast", FIELDS)
def test_level1_product_and_dinv(cuda, ne, fkind, contrast):
    """level_apply(1) torch.equal to restrict(A_0 prolong_add(x, 0)) with the index-free fine operator of the field, within
    1e-13 of each row's absolute sum of the CSR field hierarchy's level 1, and level_dinv(1) bit-identical to it."""
    import torch
    from pcg_mpi_solver_b200.hexop import HexBoxOperator
    f = _field(ne, fkind, contrast, seed=sum(ne))
    blk, op, mr, mc = _setup(cuda, f)
    info = mr.info()
    assert info["coarse"] == "rap" and info["levels"] >= 3
    A0 = HexBoxOperator(blk, device=cuda, E_field=f)
    rng = np.random.default_rng(contrast + sum(ne))
    n1 = info["n"][1]
    rp, col, val = mc.level_matrix(1)
    import scipy.sparse as sp
    A1 = sp.csr_matrix((_np(val), _np(col), _np(rp)), shape=(n1, n1))
    absA = abs(A1)
    for x in (rng.standard_normal(n1), np.ones(n1)):
        xt = _t(x, cuda)
        y = mr.level_apply(1, xt)
        ref = mr.restrict(0, A0.apply_local(mr.prolong_add(0, xt, torch.zeros(mr.n, dtype=torch.float64, device=cuda))))
        assert torch.equal(y, ref)
        err = np.abs(_np(y) - A1 @ x) / (absA @ np.abs(x))
        _stat("level-1 product vs CSR / row |A||x|", err.max())
        assert err.max() <= 1e-13, float(err.max())
    assert torch.equal(mr.level_dinv(1), mc.level_dinv(1))
    assert torch.equal(mr.level_dinv(0), mc.level_dinv(0))


@pytest.mark.parametrize("ne", [(16, 8, 12), (32, 32, 32), (64, 64, 64), (128, 128, 128)])
def test_levels_from_two_on_bit_identical_to_the_field_hierarchy(cuda, ne):
    """Levels >= 2: CSR and D^-1 bit-identical, lambda equal; lambda_1 within 1e-10.  At 128^3 level 1 has 64 element layers
    of 18.9 MB, so its matrices are built in two slabs (56 + 8 layers) under the 1 GiB cap."""
    import torch
    from pcg_mpi_solver_b200 import _lib
    f = _field(ne, "random", 100, seed=7)
    _, _, mr, mc = _setup(cuda, f, kind="hexop")
    ir, ic = mr.info(), mc.info()
    assert ir["levels"] == ic["levels"] and ir["n"] == ic["n"]
    L = ir["levels"]
    for l in range(2, L - 1):
        assert all(torch.equal(a, b) for a, b in zip(mr.level_matrix(l), mc.level_matrix(l))), l
    for l in range(2, L - 1):
        assert torch.equal(mr.level_dinv(l), mc.level_dinv(l)), l
    assert ir["lambda"][2:] == ic["lambda"][2:]
    _stat("lambda_1 relative difference", abs(ir["lambda"][1] - ic["lambda"][1]) / ic["lambda"][1])
    assert abs(ir["lambda"][1] - ic["lambda"][1]) <= 1e-10 * ic["lambda"][1]
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*no CSR"):
        mr.level_matrix(1)
    # the coarsest solve is the same factor
    r = _t(np.random.default_rng(1).standard_normal(ir["n"][-1]), cuda)
    assert torch.equal(mr.coarse_solve(r), mc.coarse_solve(r))
    sr, sc = mr.setup_info(), mc.setup_info()
    assert 0 < sr["element_matrix_peak_bytes"] and sr["galerkin_ms"] > 0
    from pcg_mpi_solver_b200.multigrid import rap_setup_peak_bytes
    assert sr["element_matrix_peak_bytes"] == rap_setup_peak_bytes(ne)
    if ne[0] == 128:
        assert sr["element_matrix_peak_bytes"] < sc["element_matrix_peak_bytes"]


def test_repeated_create_is_bit_identical(cuda):
    import torch
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    f = _field((32, 16, 16), "inclusion", 100)
    blk, op, mr, _ = _setup(cuda, f, both=False)
    m2 = HexMultigrid(op, blk, E_field=f, coarse="rap")
    assert mr.info() == m2.info()
    for l in range(mr.info()["levels"] - 1):
        assert torch.equal(mr.level_dinv(l), m2.level_dinv(l))
    r = _t(np.random.default_rng(5).standard_normal(mr.n), cuda)
    assert torch.equal(mr.apply(r), m2.apply(r))


@pytest.mark.parametrize("degree", [1, 2, 3])
@pytest.mark.parametrize("kind", ["csr", "ebe_ordered", "hexop"])
def test_vcycle_against_the_field_hierarchy(cuda, kind, degree):
    """Within 1e-12 of the CSR field hierarchy's V-cycle and symmetric to 1e-12, on CSR, ordered EBE and index-free fine
    operators."""
    for ne, contrast in (((16, 16, 16), 100), ((16, 8, 12), 1000)):
        f = _field(ne, "inclusion", contrast, seed=degree)
        _, _, mr, mc = _setup(cuda, f, kind=kind, degree=degree)
        u, v = np.random.default_rng(10 * degree + contrast).standard_normal((2, mr.n))
        Mu, Mv = _np(mr.apply(_t(u, cuda))), _np(mr.apply(_t(v, cuda)))
        err = _rel(Mu, _np(mc.apply(_t(u, cuda))))
        _stat("V-cycle vs CSR field hierarchy", err)
        assert err <= 1e-12, (kind, degree, ne, err)
        asym = abs(np.dot(Mu, v) - np.dot(u, Mv)) / (np.linalg.norm(Mu) * np.linalg.norm(v))
        _stat("V-cycle asymmetry", asym)
        assert asym <= 1e-12, asym


def test_constant_field_matches_the_index_free_hierarchy(cuda):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    ne = (32, 16, 16)
    f = np.ones((ne[2], ne[1], ne[0]))
    blk, op, mr, _ = _setup(cuda, f, both=False)
    mi = HexMultigrid(op, blk, coarse="index_free")
    u = np.random.default_rng(2).standard_normal(mr.n)
    err = _rel(_np(mr.apply(_t(u, cuda))), _np(mi.apply(_t(u, cuda))))
    _stat("constant field vs index-free hierarchy", err)
    assert err <= 1e-11, err


@pytest.mark.parametrize("n", [32, 64, 128])
@pytest.mark.parametrize("contrast", [1, 10, 100])
def test_mg_pcg_matches_the_field_hierarchy(cuda, n, contrast):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    f = _field((n, n, n), "inclusion", contrast)
    blk, op, mr, mc = _setup(cuda, f)
    b = load_vector(blk, device=cuda)
    x, info = op.solve(b, mr, 1e-8, 500)
    xc, infoc = op.solve(b, mc, 1e-8, 500)
    assert info.flag == infoc.flag == 0, (info.flag, infoc.flag)
    _stat(f"MG-PCG |iters - CSR iters| {n}^3", abs(info.iters - infoc.iters))
    assert abs(info.iters - infoc.iters) <= 1, (info.iters, infoc.iters)
    err = float((x - xc).norm() / xc.norm())
    _stat("MG-PCG x vs CSR field hierarchy", err)
    assert err <= 1e-9, err


@pytest.mark.parametrize("n", [16, 32])
def test_mg_pcg_index_free_fine_operator_bit_identical_to_ordered(cuda, n):
    import torch
    from pcg_mpi_solver_b200.hexmesh import load_vector
    f = _field((n, n, n), "inclusion", 100)
    blk, oh, mh, _ = _setup(cuda, f, "hexop", both=False)
    _, oo, mo, _ = _setup(cuda, f, "ebe_ordered", both=False)
    assert mh.info()["lambda"] == mo.info()["lambda"]
    b = load_vector(blk, device=cuda)
    (xa, ia), (xb, ib) = (o.solve(b, m, 1e-10, 200, record_resvec=True, trace=True) for o, m in ((oh, mh), (oo, mo)))
    assert torch.equal(xa, xb) and _bits(ia.resvec, ib.resvec) and ia.iters == ib.iters and ia.flag == ib.flag == 0
    assert ia.trace_total == ib.trace_total and ia.trace.tobytes() == ib.trace.tobytes()


@pytest.mark.parametrize("use_graph", [False, True])
def test_launches_per_iteration_are_constant(cuda, use_graph):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    f = _field((32, 16, 16), "random", 10)
    blk, op, mr, _ = _setup(cuda, f, degree=3, both=False)
    b = load_vector(blk, device=cuda)
    counts = []
    for m in (4, 8, 12):
        _, info = op.solve(b, mr, 1e-30, m, fixed_iters=True, use_graph=use_graph, check_every=4)
        assert info.loop_iters == m and info.flag == 1
        counts.append(info.launches)
    assert counts[1] - counts[0] == counts[2] - counts[1] > 0, counts


def test_nan_in_minv_gives_flag_2(cuda):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    f = _field((16, 8, 8), "random", 10)
    blk, op, _, _ = _setup(cuda, f, both=False)
    minv = op.jacobi()
    minv[5] = float("nan")
    bad = HexMultigrid(op, blk, minv=minv, E_field=f, coarse="rap")
    _, info = op.solve(load_vector(blk, device=cuda), bad, 1e-8, 50)
    assert info.flag == 2


# ------------------------------------------------------------------------------------------- memory and refusals
def _free(cuda):
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(cuda)[0]


@pytest.mark.parametrize("ne", [(16, 16, 16), (16, 8, 12), (32, 32, 32), (64, 64, 64)])
def test_bytes_equal_rap_bytes(cuda, ne):
    from pcg_mpi_solver_b200.multigrid import rap_bytes
    _, _, mr, _ = _setup(cuda, _field(ne, "random", 10), both=False)
    assert mr.info()["bytes"] == rap_bytes(ne)


def test_refusals_leak_no_device_memory(cuda):
    """nu = 0.6 (an indefinite coarsest matrix, refused after the hierarchy was allocated), a non-positive Ck and bad
    arguments of the C entry point (refused before anything is allocated) give every byte back."""
    import ctypes
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, field_ck, hex_element_stiffness
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    from tests import gmg_cases as G
    ne = G.BAD_NU_BOX
    f = _field(ne, "random", 10)
    _setup(cuda, f, both=False)                       # every set-up kernel loaded before the measurement
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0], nu=G.BAD_NU)
    op = SubdomainOperator(_operator(blk, cuda, "hexop", f))
    minv = op.jacobi()
    ck = field_ck(f, blk, cuda)
    neg = -ck
    free0 = _free(cuda)
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*not positive definite"):
        HexMultigrid(op, blk, minv=minv, E_field=f, coarse="rap")
    lib = _lib.load()
    ke = np.ascontiguousarray(hex_element_stiffness(1.0, 0.3))
    kep = ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    out = ctypes.c_void_p()
    box = blk.cbox()
    part = HexBlock(tuple(2 * v for v in ne), (0, 0, 0), ne).cbox()
    for args in ((op._solver, ctypes.byref(box), kep, _lib.ptr(ck), _lib.ptr(minv), 0, 0.25),      # degree 0
                 (op._solver, ctypes.byref(box), kep, _lib.ptr(ck), _lib.ptr(minv), 2, 1.2),       # lo outside (0, 1.1)
                 (op._solver, ctypes.byref(box), kep, None, _lib.ptr(minv), 2, 0.25),              # null field
                 (op._solver, ctypes.byref(box), kep, _lib.ptr(neg), _lib.ptr(minv), 2, 0.25),     # Ck <= 0
                 (op._solver, ctypes.byref(part), kep, _lib.ptr(ck), _lib.ptr(minv), 2, 0.25),     # not the whole mesh
                 (op._solver, ctypes.byref(box), None, _lib.ptr(ck), _lib.ptr(minv), 2, 0.25)):    # null Ke
        rc = lib.pcgb_mg_create_field_rap(*args, ctypes.byref(out))
        assert rc == -1 and not out, rc
    # a box of two levels, on a solver of its size
    two = HexBlock((8, 4, 8), (0, 0, 0), (8, 4, 8), h=0.125)
    f2 = _field(two.ne, "random", 10)
    op2 = SubdomainOperator(_operator(two, cuda, "hexop", f2))
    ck2, minv2 = field_ck(f2, two, cuda), op2.jacobi()
    rc = lib.pcgb_mg_create_field_rap(op2._solver, ctypes.byref(two.cbox()), kep, _lib.ptr(ck2), _lib.ptr(minv2), 2, 0.25,
                                      ctypes.byref(out))
    assert rc == -1 and not out and b"at least 3" in lib.pcgb_last_error()
    del op2, ck2, minv2
    assert _free(cuda) >= free0


def test_level_dinv_refuses_unsmoothed_levels(cuda):
    from pcg_mpi_solver_b200 import _lib
    _, _, mr, _ = _setup(cuda, _field((16, 8, 8), "random", 10), both=False)
    for bad in (-1, mr.info()["levels"] - 1):
        with pytest.raises(_lib.PcgbError, match=r"\(-1\).*not smoothed"):
            mr.level_dinv(bad)


# ------------------------------------------------------------------------------------------- 512^3
def test_mg_pcg_on_a_512_voxel_model(cuda):
    """MG-PCG to 1e-8 on the index-free fine operator of a 512^3 inclusion field at contrast 10 (4.0e8 dofs): flag 0, the
    true relative residual (op.apply) within 1e-8, and the free-memory drop across the set-up within 1 % of rap_bytes plus
    the fine Ck field the handle keeps.  Skipped when the GPU lacks that memory, the set-up's element matrices and the
    test's own vectors."""
    import time
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, inclusion_field, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid, hex_csr_nnz, rap_bytes, rap_setup_peak_bytes
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = (512, 512, 512)
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / 512)
    n, nel = blk.n, 512 ** 3
    need = rap_bytes(ne) + rap_setup_peak_bytes(ne) + 12 * hex_csr_nnz((128,) * 3) + 8 * n * (5 + 4) + 3 * 8 * nel
    if _free(cuda) < need + (2 << 30):
        pytest.skip(f"needs {(need + (2 << 30)) / 2**30:.1f} GiB free")
    f = inclusion_field(ne, 0.4, (2.0, 6.0), 1.0, 10.0, 0)
    ft = torch.from_numpy(f).to(cuda)
    del f
    A = generate_box_operator(blk, device=cuda, E_field=ft)
    op = SubdomainOperator(A)
    minv = 1.0 / A.diagonal()
    b = load_vector(blk, device=cuda)
    free0 = _free(cuda)
    t0 = time.perf_counter()
    mg = HexMultigrid(op, blk, minv=minv, E_field=ft, coarse="rap")
    torch.cuda.synchronize()
    setup = time.perf_counter() - t0
    drop = free0 - _free(cuda)
    info = mg.info()
    assert info["bytes"] == rap_bytes(ne)
    expect = info["bytes"] + 8 * nel
    _stat("512^3 memory drop / (rap_bytes + field) - 1", abs(drop / expect - 1))
    assert abs(drop - expect) <= 0.01 * expect, (drop, expect)
    del minv, ft
    t0 = time.perf_counter()
    x, si = op.solve(b, mg, 1e-8, 300)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print(f"512^3 rap MG-PCG contrast 10: iters {si.iters} wall {wall:.2f} s set-up {setup:.2f} s bytes {info['bytes']} "
          f"drop {drop} setup_info {mg.setup_info()}")
    _stat("512^3 iterations", si.iters)
    assert si.flag == 0, (si.flag, si.iters)
    rel = float((b - op.apply(x)).norm() / b.norm())
    _stat("512^3 true relative residual", rel)
    assert rel <= 1e-8, rel


def test_zz_report_largest_errors():
    """The largest error of each kind over this module's tests (printed with -rP)."""
    for k in sorted(STATS):
        print(f"{k}: {STATS[k]:.3e}")
