"""The geometric multigrid preconditioner at its edges, against the host restatement (tests/gmg_cases.py) fed the device's
own D^-1 and lambda: the Lanczos lambda of every smoothed level, the Chebyshev smoother at degrees 1-5 and lo 0.05-0.9 on
every smoothed level, materials and spacings (with the scaling invariance M(sE) = M(E) / s), non-cubic boxes and one box
above the vector-grid cap, the coarse Cholesky solve at its 1024-thread edges and its refusal of an indefinite matrix, the
overlap refusal of pcgb_mg_apply, and MG-PCG step by step: p = fma(beta, p, M r) and the rz / #inf sums of every record
against z = M r of the snapshot residual.

Largest errors seen are collected in STATS and printed by the last test (-rP)."""
import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import gmg_cases as G
from tests import pcg_shadow as S

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -53
LD = np.longdouble
STATS = {}


def _stat(key, v):
    STATS[key] = max(STATS.get(key, 0.0), float(v))


def _setup(cuda, ne, kind="csr", degree=2, lo=0.25, E=1.0, nu=0.3, h=None, minv=None):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock(tuple(ne), (0, 0, 0), tuple(ne), h=1.0 / ne[0] if h is None else h, E=E, nu=nu)
    A = generate_matrix(blk, device=cuda) if kind == "csr" else generate_ebe(blk, device=cuda, ordered=kind == "ebe_ordered")
    op = SubdomainOperator(A)
    return blk, op, HexMultigrid(op, blk, degree=degree, lo=lo, minv=minv)


def _t(v, cuda):
    import torch
    return None if v is None else torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(cuda)


def _np(t):
    return t.cpu().numpy()


def _host(blk, mg, degree=2, lo=0.25, minv=None):
    return G.HostMultigrid(blk.ne, blk.h, degree=degree, lo=lo, lambdas=mg.info()["lambda"], minv=minv, E=blk.E, nu=blk.nu)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _check_lambdas(mg, H, minv0, key):
    """lambda of every smoothed level against the host Lanczos recurrence fed the device's D^-1: level 0 the given Minv,
    levels >= 1 1/diag at spacing 2^l h."""
    lam = mg.info()["lambda"]
    for l in range(len(H.ne) - 1):
        ref = G.lanczos_lambda(H.A[l], minv0 if l == 0 else 1.0 / H.A[l].diag)
        err = abs(lam[l] - ref) / ref
        _stat(key, err)
        assert err <= 1e-10, (l, lam[l], ref, err)


def _check_smoother(cuda, mg, H, rng, key):
    """One smoothing x += S (b - A x) from x = 0 and from x != 0 on every smoothed level: normwise and max-abs within 1e-13."""
    info = mg.info()
    for l in range(info["levels"] - 1):
        b, x0 = rng.standard_normal((2, info["n"][l]))
        for start in (np.zeros_like(x0), x0):
            x = _np(mg.smooth(l, _t(b, cuda), _t(start, cuda)))
            ref, _ = H.smooth(l, b, start, False)
            nerr, merr = _rel(x, ref), float(np.abs(x - ref).max() / np.abs(ref).max())
            _stat(key + " norm", nerr)
            _stat(key + " max", merr)
            assert nerr <= 1e-13 and merr <= 1e-13, (l, nerr, merr)


def _check_coarse(cuda, mg, Ac, r, key):
    """Coarse solve: residual within 1e-12 |r|, forward error within 2 n 2^-53 kappa_2(A) |z| of a refined host solve (the
    normwise bound of a backward-stable Cholesky solve), and a repeat bit-identical.  Returns the forward error in units of
    n 2^-53 kappa |z|."""
    import torch
    n = r.size
    zt = mg.coarse_solve(_t(r, cuda))
    z = _np(zt)
    assert np.linalg.norm(Ac @ z - r) <= 1e-12 * np.linalg.norm(r)
    ref = G.refined_solve(Ac, r)
    fwd = np.linalg.norm(z - ref) / (n * EPS * np.linalg.cond(Ac) * np.linalg.norm(ref))
    _stat(key, fwd)
    assert fwd <= 2.0, fwd
    assert torch.equal(mg.coarse_solve(_t(r, cuda)), zt)


def _check_vcycle(cuda, mg, H, rng, key, reproducible=True, bound=1e-12):
    """Whole V-cycle against the host, symmetric to 1e-12, positive on random vectors, bit-reproducible."""
    import torch
    u, v = rng.standard_normal((2, mg.n))
    Mu_t = mg.apply(_t(u, cuda))
    Mu, Mv = _np(Mu_t), _np(mg.apply(_t(v, cuda)))
    err = _rel(Mu, H.apply(u))
    _stat(key + " vs host", err)
    assert err <= bound, err
    asym = abs(np.dot(Mu, v) - np.dot(u, Mv)) / (np.linalg.norm(Mu) * np.linalg.norm(v))
    _stat(key + " asymmetry", asym)
    assert asym <= 1e-12, asym
    for w in rng.standard_normal((3, mg.n)):
        assert np.dot(_np(mg.apply(_t(w, cuda))), w) > 0
    if reproducible:
        assert torch.equal(mg.apply(_t(u, cuda)), Mu_t)


# ------------------------------------------------------------------------------------------- lambda
@pytest.mark.parametrize("kind", ["csr", "ebe_ordered", "ebe"])
def test_lambda_of_every_level_matches_the_host_recurrence(cuda, kind):
    blk, op, mg = _setup(cuda, (16, 16, 16), kind)
    _check_lambdas(mg, _host(blk, mg), _np(op.jacobi()), "lambda")


def test_lambda_and_smoother_with_a_callers_minv(cuda):
    """Minv = c jacobi: lambda_0 scales by c, the coarse lambdas stay, and the smoother is the same polynomial (to 1e-13).
    A random positive Minv: lambda_0 and the level-0 smoother against HostMultigrid(minv=...)."""
    ne, c = (16, 8, 8), 3.0
    blk, op, mg = _setup(cuda, ne)
    jac = op.jacobi()
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    mgc = HexMultigrid(op, blk, minv=c * jac)
    lam, lamc = mg.info()["lambda"], mgc.info()["lambda"]
    assert abs(lamc[0] - c * lam[0]) <= 1e-12 * c * lam[0], (lamc[0], c * lam[0])
    assert lamc[1:] == lam[1:]
    rng = np.random.default_rng(21)
    b, x0 = rng.standard_normal((2, mg.n))
    for start in (np.zeros_like(x0), x0):
        x, xc = _np(mg.smooth(0, _t(b, cuda), _t(start, cuda))), _np(mgc.smooth(0, _t(b, cuda), _t(start, cuda)))
        _stat("scaled Minv smoother", _rel(xc, x))
        assert _rel(xc, x) <= 1e-13
    minv = _np(jac) * rng.uniform(0.5, 1.5, mg.n)
    mgr = HexMultigrid(op, blk, minv=_t(minv, cuda))
    H = _host(blk, mgr, minv=minv)
    _check_lambdas(mgr, H, minv, "lambda random Minv")
    for start in (np.zeros_like(x0), x0):
        x = _np(mgr.smooth(0, _t(b, cuda), _t(start, cuda)))
        ref, _ = H.smooth(0, b, start, False)
        _stat("random Minv smoother", _rel(x, ref))
        assert _rel(x, ref) <= 1e-13


# ------------------------------------------------------------------------------------------- smoother degree and interval
@pytest.mark.parametrize("lo", [0.05, 0.25, 0.9])
@pytest.mark.parametrize("degree", [1, 2, 3, 4, 5])
def test_smoother_and_vcycle_at_every_degree_and_interval(cuda, degree, lo):
    """Degree 1 has no recurrence step; degree >= 3 runs c1[j], c2[j] for j >= 1.  The smoother on every smoothed level, and
    the whole V-cycle (host, symmetry, positivity, bit-reproducibility) on CSR and the ordered EBE operator."""
    ne = (16, 16, 16)
    rng = np.random.default_rng(100 * degree + int(100 * lo))
    for kind in ("csr", "ebe_ordered"):
        blk, op, mg = _setup(cuda, ne, kind, degree=degree, lo=lo)
        H = _host(blk, mg, degree, lo)
        if kind == "csr":
            _check_smoother(cuda, mg, H, rng, "smoother degree/lo")
        _check_vcycle(cuda, mg, H, rng, "V-cycle degree/lo")


# ------------------------------------------------------------------------------------------- materials and spacing
@pytest.mark.parametrize("E,nu,h", G.MATERIALS)
def test_materials_and_spacing(cuda, E, nu, h):
    """lambda, the smoother of every level, the coarse solve and the V-cycle against the host of the same material; scaling
    E or h by s leaves every lambda (1e-12) and gives M / s (1e-13)."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = (16, 8, 8)
    blk, op, mg = _setup(cuda, ne, E=E, nu=nu, h=h)
    H = _host(blk, mg)
    rng = np.random.default_rng(int(E * 10) + int(nu * 100))
    _check_lambdas(mg, H, _np(op.jacobi()), "lambda material")
    _check_smoother(cuda, mg, H, rng, "smoother material")
    _check_coarse(cuda, mg, G.coarsest_matrix(ne, h, E, nu), rng.standard_normal(mg.info()["n"][-1]), "coarse solve material")
    _check_vcycle(cuda, mg, H, rng, "V-cycle material")
    u = rng.standard_normal(mg.n)
    Mu, lam = _np(mg.apply(_t(u, cuda))), mg.info()["lambda"]
    s = 4.0
    for b2 in (HexBlock(ne, (0, 0, 0), ne, h=h, E=s * E, nu=nu), HexBlock(ne, (0, 0, 0), ne, h=s * h, E=E, nu=nu)):
        m2 = HexMultigrid(SubdomainOperator(generate_matrix(b2, device=cuda)), b2)
        lam2 = m2.info()["lambda"]
        assert all(abs(a - b) <= 1e-12 * b for a, b in zip(lam2[:-1], lam[:-1])), (lam2, lam)
        err = _rel(_np(m2.apply(_t(u, cuda))), Mu / s)
        _stat("scaled material M/s", err)
        assert err <= 1e-13, err


def test_mg_pcg_at_nu_045_converges_to_the_jacobi_solution(cuda):
    """MG-PCG reaches 1e-12 (flag 0).  Jacobi-PCG stagnates just above it on this box (flag 3 at relres 2.0e-12 on an
    H100), so its x is accepted with flag 3 when relres <= 1e-11."""
    from pcg_mpi_solver_b200.hexmesh import load_vector
    blk, op, mg = _setup(cuda, (16, 8, 8), E=210.0, nu=0.45)
    b = load_vector(blk, device=cuda)
    x, info = op.solve(b, mg, 1e-12, 200)
    xj, infoj = op.solve(b, op.jacobi(), 1e-12, 20000)
    assert info.flag == 0 and (infoj.flag == 0 or (infoj.flag == 3 and infoj.relres <= 1e-11)), (info.flag, infoj.flag, infoj.relres)
    err = float((x - xj).norm() / xj.norm())
    _stat("nu 0.45 MG-PCG vs Jacobi-PCG", err)
    assert err <= 1e-9, err


# ------------------------------------------------------------------------------------------- boxes
@pytest.mark.parametrize("ne", [(32, 16, 8), (24, 12, 12)])
def test_vcycle_on_non_cubic_boxes(cuda, ne):
    rng = np.random.default_rng(sum(ne))
    for kind in ("csr", "ebe_ordered", "ebe"):
        blk, op, mg = _setup(cuda, ne, kind)
        _check_vcycle(cuda, mg, _host(blk, mg), rng, "V-cycle non-cubic", reproducible=kind != "ebe")


def test_box_above_the_vector_grid_cap(cuda):
    """(96, 64, 64): 1 216 800 fine dofs, above 8 CTAs x SMs x 1024 threads, so the grid-stride loops of the smoother and
    Lanczos kernels run more than once: lambda, the fine smoother and the V-cycle against the host."""
    import torch
    ne = (96, 64, 64)
    cap = min(8 * torch.cuda.get_device_properties(cuda).multi_processor_count, 2048) * 1024
    assert 3 * G.nfree(ne) == 1216800 > cap
    blk, op, mg = _setup(cuda, ne)
    H = _host(blk, mg)
    lam = mg.info()["lambda"]
    ref = G.lanczos_lambda(H.A[0], _np(op.jacobi()))
    _stat("lambda above cap", abs(lam[0] - ref) / ref)
    assert abs(lam[0] - ref) <= 1e-10 * ref
    rng = np.random.default_rng(96)
    b, x0 = rng.standard_normal((2, mg.n))
    for start in (np.zeros_like(x0), x0):
        x = _np(mg.smooth(0, _t(b, cuda), _t(start, cuda)))
        ref, _ = H.smooth(0, b, start, False)
        _stat("smoother above cap", _rel(x, ref))
        assert _rel(x, ref) <= 1e-13
    _check_vcycle(cuda, mg, H, rng, "V-cycle above cap")


# ------------------------------------------------------------------------------------------- coarse solve
@pytest.mark.parametrize("ne", sorted(G.COARSE_SIZES))
def test_coarse_solve_at_its_cta_edges(cuda, ne):
    """Coarsest n = 54 ... 1536 (1020 | 1026 on either side of one 1024-thread pass): residual within 1e-12, forward error
    within 2 n 2^-53 kappa_2(A) |z| of a refined host solve, and a repeat bit-identical."""
    n = G.COARSE_SIZES[ne]
    blk, op, mg = _setup(cuda, ne)
    assert mg.info()["n"][-1] == n
    _check_coarse(cuda, mg, G.coarsest_matrix(ne, blk.h), np.random.default_rng(n).standard_normal(n),
                  "coarse forward error / (n eps kappa |z|)")


def test_indefinite_coarsest_matrix_is_refused_and_gives_back_its_memory(cuda):
    """nu = 0.6: the coarsest Cholesky factorisation meets a non-positive pivot after the hierarchy was allocated; the
    refusal is PCGB_ERR_ARG and every byte goes back."""
    import gc
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    ne = G.BAD_NU_BOX
    _setup(cuda, ne)     # every set-up kernel loaded before the measurement
    blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / ne[0], nu=G.BAD_NU)
    op = SubdomainOperator(generate_matrix(blk, device=cuda))
    minv = op.jacobi()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info(cuda)[0]
    with pytest.raises(_lib.PcgbError, match=r"\(-1\).*not positive definite"):
        HexMultigrid(op, blk, minv=minv)
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info(cuda)[0] >= free0


# ------------------------------------------------------------------------------------------- the overlap refusal
def test_apply_refuses_overlapping_r_and_z(cuda):
    """z = r (and any overlap of the two ranges) is refused before any launch and r is left as it was; adjacent ranges work."""
    import torch
    from pcg_mpi_solver_b200 import _lib
    _, _, mg = _setup(cuda, (8, 8, 8))
    n = mg.n
    r0 = np.random.default_rng(8).standard_normal(n)
    ref = mg.apply(_t(r0, cuda))
    buf = torch.zeros(2 * n, dtype=torch.float64, device=cuda)
    buf[:n] = _t(r0, cuda)
    keep = buf.clone()
    for lo_, hi_ in ((0, n), (n - 1, 2 * n - 1), (1, n + 1)):
        with pytest.raises(_lib.PcgbError, match=r"\(-1\).*overlap"):
            mg.apply(buf[:n], out=buf[lo_:hi_])
        torch.cuda.synchronize()
        assert torch.equal(buf, keep)
    z = mg.apply(buf[:n], out=buf[n:])
    assert torch.equal(z, ref) and torch.equal(buf[:n], keep[:n])


# ------------------------------------------------------------------------------------------- MG-PCG step by step
def _fma_close(got, a, b, c):
    """got is a*b + c rounded once, within 1 ulp plus the long-double reference's own rounding (as test_gpu_pcg_steps)."""
    ab = LD(a) * b.astype(LD)
    ref = ab + c.astype(LD)
    bound = np.spacing(np.abs(ref.astype(np.float64))) + LD(2.0 ** -62) * (np.abs(ab) + np.abs(c.astype(LD)))
    return np.all(np.abs(got.astype(LD) - ref) <= bound)


def _check_mg_steps(cuda, kind, w, x0, K, seed):
    """_check_mg_steps_on the 8^3 box's operator of `kind` and its default preconditioner."""
    blk, op, mg = _setup(cuda, (8, 8, 8), kind)
    _check_mg_steps_on(cuda, op, mg, kind != "ebe", w, x0, K, seed, kind)


def _check_mg_steps_on(cuda, op, mg, exact, w, x0, K, seed, label):
    """Runs maxiter = k = 1..K with fixed_iters: p of iteration 0 is M b bit for bit (without x0), p of every later
    iteration is fma(beta, p, M r) of the previous run's snapshot, each record's rz is sum z r w and its #inf exact.  An
    operator that is not bit-reproducible (exact False: the atomic EBE) gets the same identities to a tolerance."""
    rng = np.random.default_rng(seed)
    n = mg.n
    b = rng.standard_normal(n)
    wv = rng.uniform(0.1, 1.0, n) if w else None
    x0v = rng.standard_normal(n) if x0 else None
    wn = np.ones(n) if wv is None else wv
    prev = None
    for k in range(1, K + 1):
        x, info = op.solve(_t(b, cuda), mg, 1e-30, k, x0=_t(x0v, cuda), w=_t(wv, cuda), fixed_iters=True, trace=True, snapshot=True)
        tr, snap = info.trace, info.snapshot
        sh = S.replay(tr, 1e-30, k, n, 3, fixed_iters=True)
        assert sh.result["flag"] == info.flag and sh.result["iters"] == info.iters
        assert [int(t) for t in tr["kind"]] == [S.HEAD] + [S.ITER] * k + [S.FINAL]
        rec = tr[k]
        p, r = snap["p"].copy(), snap["r"].copy()
        if prev is None:
            if x0v is None:
                Mb = _np(mg.apply(_t(b, cuda)))
                assert np.array_equal(p, Mb) if exact else _rel(p, Mb) <= 1e-12
        else:
            beta = float(tr[k - 1]["ctrl"]["beta"])
            zprev = _np(mg.apply(_t(prev["r"], cuda)))
            if exact:
                assert _fma_close(p, beta, prev["p"], zprev), k
            else:
                err = _rel(p, beta * prev["p"] + zprev)
                _stat("MG-PCG p atomic EBE", err)
                assert err <= 1e-12, (k, err)
        z = _np(mg.apply(_t(r, cuda)))
        t = z.astype(LD) * (r.astype(LD) * wn.astype(LD))
        mag = float(np.abs(t).sum())
        dev = abs(LD(rec["inp"][S.RZ]) - t.sum())
        _stat(f"MG-PCG rz / sum|terms| {label}", float(dev) / mag)
        assert dev <= ((n + 2) * EPS if exact else 1e-12) * mag, (k, float(dev) / mag)
        assert float(rec["inp"][S.NINF]) == float((~np.isfinite(z)).sum())
        prev = {"p": p, "r": r}


@pytest.mark.parametrize("x0", [False, True])
@pytest.mark.parametrize("w", [False, True])
@pytest.mark.parametrize("kind", ["csr", "ebe_ordered", "ebe"])
def test_mg_pcg_step_by_step(cuda, kind, w, x0):
    _check_mg_steps(cuda, kind, w, x0, K=12, seed=7 + 2 * w + x0)


def test_nan_in_minv_counts_every_non_finite_z(cuda):
    """A NaN in the fine Minv: the head records #inf = the number of non-finite entries of M b for that Minv (flag 2)."""
    from pcg_mpi_solver_b200.hexmesh import load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    blk, op, _ = _setup(cuda, (16, 8, 8))
    minv = op.jacobi()
    minv[5] = float("nan")
    bad = HexMultigrid(op, blk, minv=minv)
    b = load_vector(blk, device=cuda)
    _, info = op.solve(b, bad, 1e-8, 50, trace=True)
    assert info.flag == 2
    z = _np(bad.apply(b))
    nf = int((~np.isfinite(z)).sum())
    assert nf > 0 and float(info.trace[0]["inp"][S.NINF]) == float(nf)


def test_zz_report_largest_errors():
    """The largest error of each kind over this module's tests (printed with -rP)."""
    for k in sorted(STATS):
        print(f"{k}: {STATS[k]:.3e}")
