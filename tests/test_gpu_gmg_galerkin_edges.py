"""The two Galerkin multigrid hierarchies at their edges: HexMultigrid(E_field=...) ("field", pcgb_mg_create_field) and
HexMultigrid(coarsening="any") ("any", pcgb_mg_create_any, uniform or with a field), against the host restatements
(tests/voxel_cases.py, tests/gmg_any_cases.py) fed the device's own lambda and D^-1: every level matrix against scipy
P^T A P at every material, lambda, the smoother and the V-cycle at degrees 1-5 and lo 0.05-0.9, a caller's Minv, the scaling
identities, the uniform "any" box against the same box given as a constant field, hierarchies of two materials built
interleaved (all of them read the one Ke in constant memory), the coarsest solve's forward error up to contrast 1000, the
nu = 0.6 and argument refusals, MG-PCG step by step, a NaN in Minv, the EBE operators and MG-PCG at nu = 0.45.

The checks are those of tests/test_gpu_gmg_edges.py.  Largest errors seen go into its STATS under keys naming "galerkin"
and are printed by the last test (-rP)."""
import numpy as np
import pytest
import scipy.sparse as sp

from tests import gmg_any_cases as A
from tests import gmg_cases as G
from tests import test_gpu_gmg_edges as EG
from tests import voxel_cases as V

pytestmark = pytest.mark.gpu
STATS = EG.STATS
_t, _np, _rel, _stat = EG._t, EG._np, EG._rel, EG._stat
PATHS = ["field", "any"]
# the box and field of each path's sweeps: all-even for the field path, odd and kept axes under the any rule
SWEEP = {"field": ((16, 8, 12), "random"), "any": ((25, 17, 9), "inclusion")}
# V-cycle against the host, normwise.  The whole gap is the coarsest solve: with the device's coarse_solve swapped into the
# host V-cycle the two agree to 8e-16.  The any rule's 2x2x2 coarsest matrix of a thin or odd box is far worse conditioned
# than the field path's (kappa_2 6e4 on 38x4x16 at nu = 0.45, 1.3e4 on 25x17x9, against at most 2e3), so two solves of it,
# each well inside the n 2^-53 kappa_2 forward-error bound (test_coarse_solve_forward_error), put the V-cycles up to 4.2e-12
# apart on an H100.
VCYCLE_BOUND = {"field": 1e-12, "any": 1e-11}
_BASE = {}
_SPSOLVE = {}


def _field(ne, which, scale=1.0, seed=None):
    """None (a uniform box, "any" only), a log-uniform random field or a two-phase field of contrast 10, times scale."""
    if which == "uniform":
        return None
    seed = sum(ne) if seed is None else seed
    return scale * (V.random_field(ne, seed) if which == "random" else V.two_phase(ne, 10.0, seed=seed))


def _block(ne, Em=1.0, nu=0.3, h=None):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    return HexBlock(tuple(ne), (0, 0, 0), tuple(ne), h=1.0 / ne[0] if h is None else h, E=Em, nu=nu)


def _op(cuda, blk, field, kind="csr"):
    from pcg_mpi_solver_b200.hexmesh import generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    M = generate_matrix(blk, device=cuda, E_field=field) if kind == "csr" else \
        generate_ebe(blk, device=cuda, ordered=kind == "ebe_ordered", E_field=field)
    return SubdomainOperator(M)


def _mg(op, blk, path, field, degree=2, lo=0.25, minv=None):
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    return HexMultigrid(op, blk, degree=degree, lo=lo, minv=minv, E_field=field, coarsening="any" if path == "any" else "even")


def _setup(cuda, path, ne, field, kind="csr", degree=2, lo=0.25, Em=1.0, nu=0.3, h=None, minv=None):
    blk = _block(ne, Em, nu, h)
    op = _op(cuda, blk, field, kind)
    return blk, op, _mg(op, blk, path, field, degree, lo, minv)


def _host_field(blk, field):
    return A.uniform_field(blk.ne, blk.E) if field is None else field


def _host_mats(path, blk, field):
    """The host Galerkin level matrices of the hierarchy."""
    return (V.level_matrices if path == "field" else A.level_matrices)(_host_field(blk, field), blk.h, blk.nu)


def _host(path, blk, mg, field, mats, degree=2, lo=0.25, minv=None):
    cls = V.HostFieldMultigrid if path == "field" else A.HostAnyMultigrid
    return cls(_host_field(blk, field), blk.h, degree=degree, lo=lo, lambdas=mg.info()["lambda"], minv=minv, nu=blk.nu, mats=mats)


def _ptap(path, blk, field):
    """Every level as scipy P^T A P from the host fine voxel matrix."""
    f = _host_field(blk, field)
    if path == "any":
        return A.ptap_matrices(f, blk.h, blk.nu)
    lv = G.levels_of(blk.ne)
    mats = [V.field_csr(f, blk.h, blk.nu)]
    for l in range(len(lv) - 1):
        P = G.prolongation_matrix(lv[l])
        mats.append((P.T @ mats[-1] @ P).tocsr())
    return mats


def _check_levels(mg, path, blk, field, key):
    """Every smoothed coarse level exactly symmetric and within 1e-12 of the row's largest entry of P^T A P."""
    mats = _ptap(path, blk, field)
    info = mg.info()
    assert info["n"] == [m.shape[0] for m in mats]
    for l in range(1, info["levels"] - 1):
        rp, col, val = mg.level_matrix(l)
        D = sp.csr_matrix((_np(val), _np(col), _np(rp)), shape=mats[l].shape)
        assert (D != D.T).nnz == 0, l
        diff = abs(D - mats[l]).max(axis=1).toarray().ravel()
        rowmax = abs(mats[l]).max(axis=1).toarray().ravel()
        err = float(np.max(diff / rowmax))
        _stat(key, err)
        assert err <= 1e-12, (l, err)


def _base(cuda, path):
    """The operator of the path's sweep box (built once), its field, host level matrices and Jacobi Minv."""
    if path not in _BASE:
        ne, which = SWEEP[path]
        f = _field(ne, which)
        blk = _block(ne)
        op = _op(cuda, blk, f)
        _BASE[path] = (blk, op, f, _host_mats(path, blk, f), _np(op.jacobi()))
    return _BASE[path]


# ------------------------------------------------------------------------------------------- materials and spacing
def _material_case(path, h):
    if path == "field":
        return ((16, 16, 16), "inclusion") if h == 0.125 else ((16, 8, 12), "random")
    return ((25, 17, 9), "uniform") if h == 0.125 else ((38, 4, 16), "random")


@pytest.mark.parametrize("Em,nu,h", G.MATERIALS)
@pytest.mark.parametrize("path", PATHS)
def test_materials_and_spacing(cuda, path, Em, nu, h):
    """The field (times E) or, on a uniform "any" box, block.E: level matrices against P^T A P (1e-12), lambda of every
    smoothed level against the host Lanczos (1e-10), one smoothing per level (1e-13) and the V-cycle (VCYCLE_BOUND, symmetric
    to 1e-12) against the host of the same material."""
    ne, which = _material_case(path, h)
    f = _field(ne, which, Em)
    blk, op, mg = _setup(cuda, path, ne, f, Em=Em, nu=nu, h=h)
    _check_levels(mg, path, blk, f, f"galerkin {path} level matrices vs PtAP (/ row max)")
    minv = _np(op.jacobi())
    H = _host(path, blk, mg, f, _host_mats(path, blk, f), minv=minv)
    rng = np.random.default_rng(int(Em * 10) + int(nu * 100) + int(h * 8))
    EG._check_lambdas(mg, H, minv, f"galerkin {path} lambda")
    EG._check_smoother(cuda, mg, H, rng, f"galerkin {path} smoother")
    EG._check_vcycle(cuda, mg, H, rng, f"galerkin {path} V-cycle", bound=VCYCLE_BOUND[path])


# ------------------------------------------------------------------------------------------- smoother degree and interval
@pytest.mark.parametrize("lo", [0.05, 0.25, 0.9])
@pytest.mark.parametrize("degree", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("path", PATHS)
def test_smoother_and_vcycle_at_every_degree_and_interval(cuda, path, degree, lo):
    """Degree 1 has no recurrence step, degree >= 3 runs c1[j], c2[j] for j >= 1: one smoothing per level (1e-13) and the
    V-cycle (VCYCLE_BOUND, symmetric, positive, bit-reproducible) against the host of the same degree and interval."""
    blk, op, f, mats, minv = _base(cuda, path)
    mg = _mg(op, blk, path, f, degree, lo)
    H = _host(path, blk, mg, f, mats, degree, lo, minv)
    rng = np.random.default_rng(100 * degree + int(100 * lo))
    EG._check_smoother(cuda, mg, H, rng, f"galerkin {path} smoother degree/lo")
    EG._check_vcycle(cuda, mg, H, rng, f"galerkin {path} V-cycle degree/lo", bound=VCYCLE_BOUND[path])


# ------------------------------------------------------------------------------------------- a caller's Minv
@pytest.mark.parametrize("path", PATHS)
def test_lambda_and_smoother_with_a_callers_minv(cuda, path):
    """Minv = 3 jacobi: lambda_0 scales by 3 (1e-12), the coarse lambdas are bitwise the default's, and one smoothing is the
    default one (1e-13).  A random positive Minv: lambda_0 and the level-0 smoother against the host given that Minv."""
    blk, op, f, mats, minv = _base(cuda, path)
    c = 3.0
    jac = op.jacobi()
    mg, mgc = _mg(op, blk, path, f), _mg(op, blk, path, f, minv=c * jac)
    lam, lamc = mg.info()["lambda"], mgc.info()["lambda"]
    err = abs(lamc[0] - c * lam[0]) / (c * lam[0])
    _stat(f"galerkin {path} lambda with 3 jacobi vs 3 lambda", err)
    assert err <= 1e-12, (lamc[0], c * lam[0])
    assert lamc[1:] == lam[1:]
    rng = np.random.default_rng(21)
    b, x0 = rng.standard_normal((2, mg.n))
    for start in (np.zeros_like(x0), x0):
        x, xc = _np(mg.smooth(0, _t(b, cuda), _t(start, cuda))), _np(mgc.smooth(0, _t(b, cuda), _t(start, cuda)))
        _stat(f"galerkin {path} scaled Minv smoother", _rel(xc, x))
        assert _rel(xc, x) <= 1e-13
    mr = minv * rng.uniform(0.5, 1.5, mg.n)
    mgr = _mg(op, blk, path, f, minv=_t(mr, cuda))
    H = _host(path, blk, mgr, f, mats, minv=mr)
    EG._check_lambdas(mgr, H, mr, f"galerkin {path} lambda random Minv")
    for start in (np.zeros_like(x0), x0):
        x = _np(mgr.smooth(0, _t(b, cuda), _t(start, cuda)))
        ref, _ = H.smooth(0, b, start, False)
        _stat(f"galerkin {path} random Minv smoother", _rel(x, ref))
        assert _rel(x, ref) <= 1e-13


# ------------------------------------------------------------------------------------------- scaling and the uniform box
@pytest.mark.parametrize("path", PATHS)
def test_scaling_the_modulus_by_4(cuda, path):
    """The field times 4 (both paths) and, under "any", a uniform box at E = 4 against E = 1: every lambda equal (1e-12)
    and M_4 r = (M r) / 4 (1e-13)."""
    ne, which = SWEEP[path]
    f = _field(ne, which)
    cases = [("field x4", f, 4.0 * f, 1.0, 1.0)] + ([("uniform E=4", None, None, 1.0, 4.0)] if path == "any" else [])
    u = np.random.default_rng(4).standard_normal(3 * G.nfree(ne))
    for name, f1, f4, e1, e4 in cases:
        _, _, m1 = _setup(cuda, path, ne, f1, Em=e1)
        _, _, m4 = _setup(cuda, path, ne, f4, Em=e4)
        lam1, lam4 = m1.info()["lambda"], m4.info()["lambda"]
        k = m1.info()["levels"] - 1
        lerr = max(abs(a - b) / b for a, b in zip(lam4[:k], lam1[:k]))
        _stat(f"galerkin scaling lambda ({path} {name})", lerr)
        assert lerr <= 1e-12, (lam4, lam1)
        err = _rel(_np(m4.apply(_t(u, cuda))), _np(m1.apply(_t(u, cuda))) / 4.0)
        _stat(f"galerkin scaling M/4 ({path} {name})", err)
        assert err <= 1e-13, err


def test_uniform_any_box_equals_the_constant_field(cuda):
    """A uniform box at E = c under "any" and the same operator's "any" hierarchy with np.full(c): both make Ck = c h as
    the same double product, so the level matrices, lambda and the V-cycle are bit for bit the same."""
    import torch
    ne, c = (25, 17, 9), 7.5
    blk = _block(ne, Em=c)
    op = _op(cuda, blk, None)
    mu, mf = _mg(op, blk, "any", None), _mg(op, blk, "any", A.uniform_field(ne, c))
    assert mu.info()["lambda"] == mf.info()["lambda"]
    for l in range(1, mu.info()["levels"] - 1):
        assert all(torch.equal(a, b) for a, b in zip(mu.level_matrix(l), mf.level_matrix(l))), l
    r = _t(np.random.default_rng(7).standard_normal(mu.n), cuda)
    assert torch.equal(mu.apply(r), mf.apply(r))


def test_interleaved_materials_each_get_their_own_ke(cuda):
    """Operators A (nu = 0.2) and B (nu = 0.45) first, then field, field, any, any hierarchies of A, B, A, B: each against
    P^T A P of its own material.  The fine fill and the level-1 Galerkin kernels read the one Ke in constant memory, so a
    hierarchy that did not upload its own would take B's."""
    ne = (16, 8, 12)
    f = _field(ne, "random")
    blocks = {nu: _block(ne, nu=nu) for nu in (0.2, 0.45)}
    ops = {nu: _op(cuda, blocks[nu], f) for nu in (0.2, 0.45)}
    for path, nu in (("field", 0.2), ("field", 0.45), ("any", 0.2), ("any", 0.45)):
        mg = _mg(ops[nu], blocks[nu], path, f)
        _check_levels(mg, path, blocks[nu], f, f"galerkin {path} interleaved level matrices vs PtAP (/ row max)")


# ------------------------------------------------------------------------------------------- coarse solve
COARSE_CASES = [("field", ne) for ne in sorted(G.COARSE_SIZES)] + [("any", (25, 17, 9)), ("any", (38, 4, 16))]


@pytest.mark.parametrize("path,ne", COARSE_CASES)
def test_coarse_solve_forward_error(cuda, path, ne):
    """A random field of contrast 1 ... 1000; the coarsest solve against the host Galerkin coarsest matrix: residual within
    1e-12 |r|, forward error within 2 n 2^-53 kappa_2(A) |z| of a refined host solve, and a repeat bit-identical."""
    f = V.random_field(ne, seed=sum(ne), lo=1.0, hi=1000.0)
    blk, op, mg = _setup(cuda, path, ne, f)
    Ac = _host_mats(path, blk, f)[-1].toarray()
    n = Ac.shape[0]
    assert mg.info()["n"][-1] == n and (path == "any" or n == G.COARSE_SIZES[ne])
    EG._check_coarse(cuda, mg, Ac, np.random.default_rng(n).standard_normal(n), f"galerkin {path} coarse forward error / (n eps kappa |z|)")


# ------------------------------------------------------------------------------------------- refusals
def _free(cuda):
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(cuda)[0]


@pytest.mark.parametrize("path,uniform", [("field", False), ("any", True), ("any", False)])
def test_indefinite_coarsest_matrix_is_refused_and_gives_back_its_memory(cuda, path, uniform):
    """nu = 0.6 on the boxes whose host Galerkin coarsest matrix is indefinite (test_gmg_galerkin_cpu.py): the coarse
    Cholesky factorisation meets a non-positive pivot after the hierarchy was allocated; PCGB_ERR_ARG and every byte back."""
    from pcg_mpi_solver_b200 import _lib
    ne = A.BAD_NU_FIELD_BOX if path == "field" else A.BAD_NU_ANY_BOX
    f = None if uniform else V.random_field(ne, seed=sum(ne))
    _setup(cuda, path, ne, f)     # every set-up kernel loaded before the measurement
    blk = _block(ne, nu=G.BAD_NU)
    op = _op(cuda, blk, f)
    minv = op.jacobi()
    free0 = _free(cuda)
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*not positive definite"):
        _mg(op, blk, path, f, minv=minv)
    assert _free(cuda) >= free0


@pytest.mark.parametrize("path", PATHS)
def test_argument_refusals_allocate_nothing(cuda, path):
    """lo 0, 1.1 or NaN and degree 0: PCGB_ERR_ARG before anything is allocated."""
    from pcg_mpi_solver_b200 import _lib
    blk, op, f, _, _ = _base(cuda, path)
    minv = op.jacobi()
    for degree, lo in ((2, 0.0), (2, 1.1), (2, float("nan")), (0, 0.25)):
        free0 = _free(cuda)
        with pytest.raises(_lib.PcgbError, match=r"\(-1\)"):
            _mg(op, blk, path, f, degree=degree, lo=lo, minv=minv)
        assert _free(cuda) >= free0, (degree, lo)


# ------------------------------------------------------------------------------------------- MG-PCG step by step
STEP_BOXES = {"field": (8, 8, 8), "any": (9, 7, 5)}


@pytest.mark.parametrize("x0", [False, True])
@pytest.mark.parametrize("w", [False, True])
@pytest.mark.parametrize("path", PATHS)
def test_mg_pcg_step_by_step(cuda, path, w, x0):
    """CSR and a random field: p_0 = M b bit for bit, then fma(beta, p, M r) within 1 ulp, rz within (n + 2) 2^-53
    sum|terms| and #inf exact on every one of 12 iterations (test_gpu_gmg_edges' identities)."""
    ne = STEP_BOXES[path]
    _, op, mg = _setup(cuda, path, ne, V.random_field(ne, seed=3))
    EG._check_mg_steps_on(cuda, op, mg, True, w, x0, 12, 7 + 2 * w + x0, f"galerkin {path}")


@pytest.mark.parametrize("path", PATHS)
def test_nan_in_minv_counts_every_non_finite_z(cuda, path):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from tests import pcg_shadow as S
    blk, op, f, _, _ = _base(cuda, path)
    minv = op.jacobi()
    minv[5] = float("nan")
    bad = _mg(op, blk, path, f, minv=minv)
    b = load_vector(blk, device=cuda)
    _, info = op.solve(b, bad, 1e-8, 50, trace=True)
    assert info.flag == 2
    z = _np(bad.apply(b))
    nf = int((~np.isfinite(z)).sum())
    assert nf > 0 and float(info.trace[0]["inp"][S.NINF]) == float(nf)


# ------------------------------------------------------------------------------------------- fine EBE operators
@pytest.mark.parametrize("kind", ["ebe_ordered", "ebe"])
@pytest.mark.parametrize("path", PATHS)
def test_vcycle_on_ebe_operators(cuda, path, kind):
    """E = 210, nu = 0.45 on the EBE operators: the V-cycle against the host (VCYCLE_BOUND), symmetric (1e-12);
    bit-reproducible on the ordered one."""
    ne, which = SWEEP[path]
    f = _field(ne, which, 210.0)
    blk, op, mg = _setup(cuda, path, ne, f, kind=kind, nu=0.45)
    H = _host(path, blk, mg, f, _host_mats(path, blk, f), minv=_np(op.jacobi()))
    EG._check_vcycle(cuda, mg, H, np.random.default_rng(45), f"galerkin {path} V-cycle {kind}", reproducible=kind != "ebe",
                     bound=VCYCLE_BOUND[path])


# ------------------------------------------------------------------------------------------- MG-PCG at nu = 0.45
@pytest.mark.parametrize("path", PATHS)
def test_mg_pcg_at_nu_045(cuda, path):
    """24^3 two-phase at contrast 100, nu = 0.45: flag 0 at 1e-8; the 1e-11 solution, refined once by an MG-PCG solve of its
    residual, within 1e-9 of a sparse direct solve."""
    import scipy.sparse.linalg as sla
    from pcg_mpi_solver_b200.hexmesh import load_vector
    ne = (24, 24, 24)
    f = V.two_phase(ne, 100.0, seed=24, radii=(1.0, 3.0))
    blk, op, mg = _setup(cuda, path, ne, f, nu=0.45)
    b = load_vector(blk, device=cuda)
    _, info = op.solve(b, mg, 1e-8, 300)
    assert info.flag == 0, (info.flag, info.iters)
    x, i11 = op.solve(b, mg, 1e-11, 800)
    assert i11.flag in (0, 3) and i11.relres <= 1e-10, (i11.flag, i11.relres)
    d, idd = op.solve(b - op.apply(x), mg, 1e-11, 800)
    assert idd.flag in (0, 3) and idd.relres <= 1e-10, (idd.flag, idd.relres)
    x = _np(x + d)
    if "xr" not in _SPSOLVE:
        _SPSOLVE["xr"] = sla.spsolve(V.field_csr(f, blk.h, 0.45).tocsc(), _np(b))
    err = _rel(x, _SPSOLVE["xr"])
    _stat(f"galerkin nu 0.45 MG-PCG vs spsolve ({path})", err)
    assert err <= 1e-9, err


def test_zz_report_largest_errors():
    """The largest error of each kind over this module's tests (printed with -rP)."""
    for k in sorted(STATS):
        if "galerkin" in k:
            print(f"{k}: {STATS[k]:.3e}")
