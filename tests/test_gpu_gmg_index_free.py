"""The multigrid preconditioner with index-free coarse levels (HexMultigrid(coarse="index_free"),
pcgb_mg_create_index_free): every smoothed coarse level against the index-free operator of its own box bit for bit (product
and D^-1), lambda / smoother / V-cycle against the host restatement (tests/gmg_cases.py) fed the device's lambda, the
V-cycle and MG-PCG against the CSR hierarchy of the same box, determinism, the launch count of an iteration, the refusals,
and MG-PCG on a 512^3 box when the GPU has the memory.

Largest errors seen are collected in STATS and printed by the last test (-rP)."""
import numpy as np
import pytest

from tests import gmg_cases as G
from tests import pcg_shadow as S

pytestmark = pytest.mark.gpu
STATS = {}


def _stat(key, v):
    STATS[key] = max(STATS.get(key, 0.0), float(v))


def _t(v, cuda):
    import torch
    return None if v is None else torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _np(t):
    return t.cpu().numpy()


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def _operator(blk, cuda, kind):
    from pcg_mpi_solver_b200.hexmesh import generate_box_operator, generate_ebe, generate_matrix
    if kind == "csr":
        return generate_matrix(blk, device=cuda)
    if kind == "hexop":
        return generate_box_operator(blk, device=cuda)
    return generate_ebe(blk, device=cuda, ordered=True)


def _setup(cuda, ne, kind="hexop", coarse="index_free", degree=2, lo=0.25, E=1.0, nu=0.3, h=None):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock(tuple(ne), (0, 0, 0), tuple(ne), h=1.0 / ne[0] if h is None else h, E=E, nu=nu)
    op = SubdomainOperator(_operator(blk, cuda, kind))
    return blk, op, HexMultigrid(op, blk, degree=degree, lo=lo, coarse=coarse)


def _host(blk, mg, degree=2, lo=0.25):
    return G.HostMultigrid(blk.ne, blk.h, degree=degree, lo=lo, lambdas=mg.info()["lambda"], E=blk.E, nu=blk.nu)


def _level_block(blk, l):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    ne = tuple(v >> l for v in blk.ne)
    return HexBlock(ne, (0, 0, 0), ne, h=blk.h * 2 ** l, E=blk.E, nu=blk.nu)


def _check_levels(cuda, blk, seed):
    """level_apply of every smoothed coarse level bit-identical to HexBoxOperator of the level's box (h = 2^l h), and D^-1
    bit-identical to 1 / its diagonal(): a degree-1 smoothing of b = 1 from x = 0 is inv_theta * (D^-1 * 1), with inv_theta
    the host's restatement of the device's Chebyshev centre."""
    import torch
    from pcg_mpi_solver_b200.hexop import HexBoxOperator
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    op = SubdomainOperator(_operator(blk, cuda, "hexop"))
    mg = HexMultigrid(op, blk, degree=1, coarse="index_free")
    info = mg.info()
    assert info["coarse"] == "index_free" and info["levels"] >= 3
    rng = np.random.default_rng(seed)
    for l in range(1, info["levels"] - 1):
        ref_op = HexBoxOperator(_level_block(blk, l), device=cuda)
        x = _t(rng.standard_normal(info["n"][l]), cuda)
        assert torch.equal(mg.level_apply(l, x), ref_op.apply_local(x)), l
        inv_theta, _, _ = G.cheb_coeffs(info["lambda"][l], 1, mg.lo)
        ones = torch.ones(info["n"][l], dtype=torch.float64, device=cuda)
        got = _np(mg.smooth(l, ones, torch.zeros_like(ones)))
        want = inv_theta * (1.0 / _np(ref_op.diagonal()))
        assert _bits(got, want), (l, float(np.abs(got - want).max()))


# ------------------------------------------------------------------------------------------- coarse products and D^-1
@pytest.mark.parametrize("E,nu,h", G.MATERIALS)
def test_coarse_levels_bit_identical_to_their_box_operator_materials(cuda, E, nu, h):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    ne = (16, 8, 8)
    _check_levels(cuda, HexBlock(ne, (0, 0, 0), ne, h=h, E=E, nu=nu), int(E) + int(100 * nu))


# level 1 at nxf = 30 / 32 / 34 and 62 / 64 / 66: the 32-node brick edge from both sides (a smoothed level halves again, so
# its widths are even; the odd ones end a hierarchy as its coarsest level, which is not an operator)
@pytest.mark.parametrize("nx", [60, 64, 68, 124, 128, 132])
def test_coarse_levels_bit_identical_at_the_brick_width(cuda, nx):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    ne = (nx, 8, 8)
    _check_levels(cuda, HexBlock(ne, (0, 0, 0), ne, h=1.0 / nx), nx)


def test_level_csr_refuses_an_index_free_level_and_level_apply_its_edges(cuda):
    import torch
    from pcg_mpi_solver_b200 import _lib
    blk, op, mg = _setup(cuda, (16, 8, 8))
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*index-free"):
        mg.level_matrix(1)
    n = mg.info()["n"]
    for bad in (0, len(n) - 1):
        with pytest.raises(_lib.PcgbError, match=r"\(-1\)"):
            mg.level_apply(bad, torch.zeros(n[bad], dtype=torch.float64, device=cuda))
    x = torch.zeros(2 * n[1], dtype=torch.float64, device=cuda)
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*overlap"):
        mg.level_apply(1, x[:n[1]], out=x[1:n[1] + 1])
    # the CSR hierarchy's level_apply is its SpMV: the CSR product of the same level, to rounding
    _, _, mc = _setup(cuda, (16, 8, 8), coarse="csr")
    assert mc.info()["coarse"] == "csr"
    v = _t(np.random.default_rng(3).standard_normal(n[1]), cuda)
    assert _rel(_np(mc.level_apply(1, v)), _np(mg.level_apply(1, v))) <= 1e-14


# ------------------------------------------------------------------------------------------- lambda, smoother, V-cycle
@pytest.mark.parametrize("lo", [0.05, 0.25, 0.9])
@pytest.mark.parametrize("degree", [1, 2, 3, 4, 5])
def test_lambda_smoother_and_vcycle_against_the_host(cuda, degree, lo):
    """On CSR, ordered EBE and index-free fine operators: lambda of every smoothed level within 1e-10 of the host Lanczos
    recurrence fed the device's D^-1 (1 / diag at spacing 2^l h), one smoothing within 1e-13, the V-cycle within 1e-12 of
    the host and symmetric to 1e-12, and within 1e-12 of the CSR hierarchy of the same box."""
    import torch
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    ne = (16, 16, 16)
    rng = np.random.default_rng(100 * degree + int(100 * lo))
    for kind in ("csr", "ebe_ordered", "hexop"):
        blk, op, mg = _setup(cuda, ne, kind, degree=degree, lo=lo)
        H = _host(blk, mg, degree, lo)
        lam = mg.info()["lambda"]
        jac = _np(op.jacobi())
        H.dinv[0] = jac
        for l in range(len(H.ne) - 1):
            ref = G.lanczos_lambda(H.A[l], jac if l == 0 else 1.0 / H.A[l].diag)
            _stat("lambda", abs(lam[l] - ref) / ref)
            assert abs(lam[l] - ref) <= 1e-10 * ref, (kind, l, lam[l], ref)
        for l in range(len(H.ne) - 1):
            b, x0 = rng.standard_normal((2, mg.info()["n"][l]))
            for start in (np.zeros_like(x0), x0):
                x = _np(mg.smooth(l, _t(b, cuda), _t(start, cuda)))
                ref, _ = H.smooth(l, b, start, False)
                _stat("smoother", _rel(x, ref))
                assert _rel(x, ref) <= 1e-13, (kind, l, _rel(x, ref))
        u, v = rng.standard_normal((2, mg.n))
        Mu_t = mg.apply(_t(u, cuda))
        Mu, Mv = _np(Mu_t), _np(mg.apply(_t(v, cuda)))
        err = _rel(Mu, H.apply(u))
        _stat("V-cycle vs host", err)
        assert err <= 1e-12, (kind, err)
        asym = abs(np.dot(Mu, v) - np.dot(u, Mv)) / (np.linalg.norm(Mu) * np.linalg.norm(v))
        _stat("V-cycle asymmetry", asym)
        assert asym <= 1e-12, asym
        assert torch.equal(mg.apply(_t(u, cuda)), Mu_t)
        mc = HexMultigrid(op, blk, degree=degree, lo=lo)
        err = _rel(Mu, _np(mc.apply(_t(u, cuda))))
        _stat("V-cycle vs CSR hierarchy", err)
        assert err <= 1e-12, (kind, err)


@pytest.mark.parametrize("E,nu,h", G.MATERIALS)
def test_vcycle_materials_against_the_host_and_the_csr_hierarchy(cuda, E, nu, h):
    ne = (16, 8, 8)
    blk, op, mg = _setup(cuda, ne, "hexop", E=E, nu=nu, h=h)
    _, _, mc = _setup(cuda, ne, "hexop", coarse="csr", E=E, nu=nu, h=h)
    u = np.random.default_rng(int(E) + int(100 * nu)).standard_normal(mg.n)
    Mu = _np(mg.apply(_t(u, cuda)))
    err = _rel(Mu, _host(blk, mg).apply(u))
    _stat("V-cycle material vs host", err)
    assert err <= 1e-12, err
    err = _rel(Mu, _np(mc.apply(_t(u, cuda))))
    _stat("V-cycle material vs CSR hierarchy", err)
    assert err <= 1e-12, err


# ------------------------------------------------------------------------------------------- MG-PCG
@pytest.mark.parametrize("n", [16, 32, 64, 128])
def test_mg_pcg_matches_the_csr_hierarchy(cuda, n):
    """On the index-free fine operator: the iteration count of the CSR hierarchy (+-1 reported in STATS) and x within 1e-9
    of it."""
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blk, op, mg = _setup(cuda, (n, n, n))
    mc = HexMultigrid(op, blk)
    b = load_vector(blk, device=cuda)
    x, info = op.solve(b, mg, 1e-8, 200)
    xc, infoc = op.solve(b, mc, 1e-8, 200)
    assert info.flag == infoc.flag == 0, (info.flag, infoc.flag)
    _stat(f"MG-PCG |iters - CSR iters| {n}^3", abs(info.iters - infoc.iters))
    assert info.iters == infoc.iters, (info.iters, infoc.iters)
    err = float((x - xc).norm() / xc.norm())
    _stat("MG-PCG x vs CSR hierarchy", err)
    assert err <= 1e-9, err


@pytest.mark.parametrize("n", [16, 32, 64])
def test_mg_pcg_on_the_index_free_fine_operator_bit_identical_to_ordered(cuda, n):
    """x, resvec and trace of MG-PCG on the index-free fine operator equal the same hierarchy on the ordered EBE operator."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import load_vector
    blk, oh, mh = _setup(cuda, (n, n, n), "hexop")
    _, oo, mo = _setup(cuda, (n, n, n), "ebe_ordered")
    assert mh.info()["lambda"] == mo.info()["lambda"]
    b = load_vector(blk, device=cuda)
    (xa, ia), (xb, ib) = (o.solve(b, m, 1e-10, 200, record_resvec=True, trace=True) for o, m in ((oh, mh), (oo, mo)))
    assert torch.equal(xa, xb) and _bits(ia.resvec, ib.resvec) and ia.iters == ib.iters and ia.flag == ib.flag == 0
    assert ia.trace_total == ib.trace_total and ia.trace.tobytes() == ib.trace.tobytes()


# ------------------------------------------------------------------------------------------- determinism
def test_repeated_create_is_bit_identical(cuda):
    import torch
    blk, op, mg = _setup(cuda, (32, 16, 16))
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    m2 = HexMultigrid(op, blk, coarse="index_free")
    assert mg.info() == m2.info()
    r = _t(np.random.default_rng(5).standard_normal(mg.n), cuda)
    assert torch.equal(mg.apply(r), m2.apply(r))


def test_nan_in_minv_counts_every_non_finite_z(cuda):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blk, op, _ = _setup(cuda, (16, 8, 8))
    minv = op.jacobi()
    minv[5] = float("nan")
    bad = HexMultigrid(op, blk, minv=minv, coarse="index_free")
    b = load_vector(blk, device=cuda)
    _, info = op.solve(b, bad, 1e-8, 50, trace=True)
    assert info.flag == 2
    nf = int((~np.isfinite(_np(bad.apply(b)))).sum())
    assert nf > 0 and float(info.trace[0]["inp"][S.NINF]) == float(nf)


def iteration_launches(levels, degree):
    """Launches of one MG-PCG iteration on the index-free fine operator with index-free coarse levels (trace off): the
    p-update, p.q reduction, fused update and norms reduction, the fine product and its p.q dot, k_mg_rz, and the V-cycle:
    per smoothed level a first Chebyshev step, restriction, prolongation and 2 degree (product + step), then the coarse
    solve."""
    return 4 + 2 + 1 + 1 + (levels - 1) * (3 + 4 * degree)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("ne,degree", [((8, 8, 8), 2), ((32, 16, 16), 3)])
def test_launches_per_iteration_are_constant(cuda, ne, degree, use_graph):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    blk, op, mg = _setup(cuda, ne, degree=degree)
    b = load_vector(blk, device=cuda)
    counts = []
    for m in (4, 8, 12):
        _, info = op.solve(b, mg, 1e-30, m, fixed_iters=True, use_graph=use_graph, check_every=4)
        assert info.loop_iters == m and info.flag == 1
        counts.append(info.launches)
    per = iteration_launches(mg.info()["levels"], degree)
    assert counts[1] - counts[0] == counts[2] - counts[1] == 4 * per, (counts, per)


# ------------------------------------------------------------------------------------------- refusals
def _free(cuda):
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(cuda)[0]


def test_refusals_leak_no_device_memory(cuda):
    """nu = 0.6 (an indefinite coarsest matrix, refused after the hierarchy was allocated) and bad arguments of the C entry
    point (refused before anything is allocated) give every byte back."""
    import ctypes
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_element_stiffness
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = G.BAD_NU_BOX
    _setup(cuda, ne)                 # every set-up kernel loaded before the measurement
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0], nu=G.BAD_NU)
    op = SubdomainOperator(_operator(blk, cuda, "hexop"))
    minv = op.jacobi()
    free0 = _free(cuda)
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*not positive definite"):
        HexMultigrid(op, blk, minv=minv, coarse="index_free")
    lib = _lib.load()
    ke = np.ascontiguousarray(hex_element_stiffness(1.0, 0.3))
    kep = ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    out = ctypes.c_void_p()
    odd = HexBlock((9, 8, 8), (0, 0, 0), (9, 8, 8)).cbox()
    part = HexBlock((16, 8, 8), (8, 0, 0), (8, 8, 8)).cbox()
    box = blk.cbox()
    for args in ((op._solver, ctypes.byref(box), kep, 1.0, 0.125, _lib.ptr(minv), 0, 0.25),        # degree 0
                 (op._solver, ctypes.byref(box), kep, 1.0, 0.125, _lib.ptr(minv), 2, 1.2),         # lo outside (0, 1.1)
                 (op._solver, ctypes.byref(box), kep, -1.0, 0.125, _lib.ptr(minv), 2, 0.25),       # E <= 0
                 (op._solver, ctypes.byref(odd), kep, 1.0, 0.125, _lib.ptr(minv), 2, 0.25),        # size / coarsening
                 (op._solver, ctypes.byref(part), kep, 1.0, 0.125, _lib.ptr(minv), 2, 0.25),       # not the whole mesh
                 (op._solver, ctypes.byref(box), None, 1.0, 0.125, _lib.ptr(minv), 2, 0.25)):      # null Ke
        rc = lib.pcgb_mg_create_index_free(*args, ctypes.byref(out))
        assert rc == -1 and not out, rc
    assert _free(cuda) >= free0


# ------------------------------------------------------------------------------------------- 512^3
def test_mg_pcg_on_a_512_cube(cuda):
    """MG-PCG to 1e-8 on the index-free fine operator of a 512^3 box (4.0e8 dofs): flag 0 in at most 16 iterations, the
    true relative residual (op.apply) within 1.1e-8, and the device memory the set-up takes within 5 % of
    index_free_bytes plus the solver's five vectors.  Skipped when the GPU lacks that memory plus the test's own vectors."""
    import time
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid, index_free_bytes
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = (512, 512, 512)
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / 512)
    n = blk.n
    need = index_free_bytes(ne) + 8 * n * (5 + 4)      # + solver vectors + minv, b, x, A x
    if _free(cuda) < need + (2 << 30):
        pytest.skip(f"needs {(need + (2 << 30)) / 2**30:.1f} GiB free")
    A = generate_box_operator(blk, device=cuda)
    minv = 1.0 / A.diagonal()
    b = load_vector(blk, device=cuda)
    free0 = _free(cuda)
    t0 = time.perf_counter()
    op = SubdomainOperator(A)
    mg = HexMultigrid(op, blk, minv=minv, coarse="index_free")
    torch.cuda.synchronize()
    setup = time.perf_counter() - t0
    drop = free0 - _free(cuda)
    info = mg.info()
    assert info["bytes"] == index_free_bytes(ne)
    expect = info["bytes"] + 5 * 8 * n
    _stat("512^3 memory drop / (bytes + solver vectors) - 1", abs(drop / expect - 1))
    assert abs(drop - expect) <= 0.05 * expect, (drop, expect)
    del minv
    t0 = time.perf_counter()
    x, si = op.solve(b, mg, 1e-8, 100)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print(f"512^3 index-free MG-PCG: iters {si.iters} wall {wall:.2f} s set-up {setup:.2f} s bytes {info['bytes']} drop {drop}")
    _stat("512^3 iterations", si.iters)
    assert si.flag == 0 and si.iters <= 16, (si.flag, si.iters)
    rel = float((b - op.apply(x)).norm() / b.norm())
    _stat("512^3 true relative residual", rel)
    assert rel <= 1.1e-8, rel


def test_zz_report_largest_errors():
    """The largest error of each kind over this module's tests (printed with -rP)."""
    for k in sorted(STATS):
        print(f"{k}: {STATS[k]:.3e}")
