"""Voxel models on the host: the element-level Galerkin product of tests/voxel_cases.py against scipy P^T A P, the constant
field against rediscretisation, hexmesh's field helpers, and host MG-PCG against host Jacobi-PCG over the contrast range."""
import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import gmg_cases as G
from tests import voxel_cases as V


@pytest.mark.parametrize("ne", [(8, 8, 8), (8, 4, 6), (16, 8, 8), (12, 8, 4)])
def test_galerkin_elements_equal_ptap(ne):
    """Assembled and clamped, the element Galerkin matrices of every coarse level equal P^T A P of the level below (P of
    gmg_cases, the kernels' transfers) to 1e-13 of the largest entry, on random log-uniform fields."""
    f = V.random_field(ne, seed=sum(ne))
    mats = V.level_matrices(f, 1.0 / ne[0])
    lv = G.levels_of(ne)
    assert len(mats) == len(lv) >= 2
    for l in range(len(lv) - 1):
        P = G.prolongation_matrix(lv[l])
        ptap = (P.T @ mats[l] @ P).tocsr()
        scale = abs(mats[l + 1]).max()
        assert abs(ptap - mats[l + 1]).max() <= 1e-13 * scale, (ne, l)
    if ne in ((8, 8, 8), (16, 8, 8)):
        assert len(lv) == 3        # two coarse levels: the second built from Galerkin element matrices


@pytest.mark.parametrize("E", [1.0, 7.5])
def test_constant_field_equals_rediscretisation(E):
    ne, h = (8, 8, 8), 1.0 / 8
    mats = V.level_matrices(np.full(ne, E), h)
    for l, nl in enumerate(G.levels_of(ne)):
        ref = R.hex_box_csr(nl, (0, 0, 0), nl, E=E, h=h * 2 ** l)
        assert abs(mats[l] - ref).max() <= 1e-13 * abs(ref).max(), l


def test_child_weights_are_trilinear_and_exact():
    """Q_c's rows sum to 1 (partition of unity), every weight is k/8 exactly, and on the coarse corners (p in {0, 2}^3) the
    interpolation is the identity."""
    for c in range(8):
        Qc = V.child_Q(c)
        assert np.array_equal(Qc.sum(axis=1), np.ones(24))
        assert np.array_equal(Qc * 8, np.round(Qc * 8))
        for l in range(8):
            p = [((c >> a) & 1) + ((l >> a) & 1) for a in range(3)]
            if all(v in (0, 2) for v in p):
                k = sum((v // 2) << a for a, v in enumerate(p))
                assert V.child_weight(c, l, k) == 1.0


def test_inclusion_field():
    from pcg_mpi_solver_b200.hexmesh import inclusion_field
    a = inclusion_field((32, 24, 16), 0.4, (2.0, 6.0), 3.0, 300.0, seed=7)
    b = inclusion_field((32, 24, 16), 0.4, (2.0, 6.0), 3.0, 300.0, seed=7)
    c = inclusion_field((32, 24, 16), 0.4, (2.0, 6.0), 3.0, 300.0, seed=8)
    assert a.shape == (16, 24, 32) and a.dtype == np.float64
    assert a.tobytes() == b.tobytes() and a.tobytes() != c.tobytes()
    assert set(np.unique(a)) == {3.0, 300.0}
    frac = float((a == 300.0).mean())
    sphere = 4.0 / 3.0 * np.pi * 6.0 ** 3 / a.size       # drawing stops within one sphere of the target
    assert 0.4 <= frac <= 0.4 + sphere, frac
    for f in (0.1, 0.25):
        g = inclusion_field((24, 24, 24), f, (1.0, 3.0), 1.0, 2.0, seed=1)
        assert f <= float((g == 2.0).mean()) <= f + 4.0 / 3.0 * np.pi * 27 / g.size
    with pytest.raises(ValueError):
        inclusion_field((8, 8, 8), 1.0, (1.0, 2.0), 1.0, 2.0, seed=0)


def test_block_field_tiles_the_global_field():
    from pcg_mpi_solver_b200.hexmesh import block_field, partition_blocks
    f = V.random_field((8, 6, 4), seed=2)
    blocks = partition_blocks((8, 6, 4), (2, 1, 2))
    out = np.zeros_like(f)
    for b in blocks:
        s = block_field(f, b)
        assert s.shape == (b.ne[2], b.ne[1], b.ne[0]) and s.flags["C_CONTIGUOUS"]
        out[b.e0[2]:b.e0[2] + b.ne[2], b.e0[1]:b.e0[1] + b.ne[1], b.e0[0]:b.e0[0] + b.ne[0]] += s
    assert np.array_equal(out, f)
    with pytest.raises(ValueError):
        block_field(f[:, :, :3], blocks[0])


def test_hex_mdf_model_carries_the_field_in_element_order():
    from pcg_mpi_solver_b200.hexmesh import hex_mdf_model, hex_type_group, HexBlock
    ng, h = (6, 4, 5), 0.25
    f = V.random_field(ng, seed=3)
    m = hex_mdf_model(ng, h=h, E_field=f)
    nodes = m.node_flat.reshape(-1, 8).astype(np.int64)
    gx = nodes[:, 0] % (ng[0] + 1)
    gy = (nodes[:, 0] // (ng[0] + 1)) % (ng[1] + 1)
    gz = nodes[:, 0] // ((ng[0] + 1) * (ng[1] + 1))
    assert np.array_equal(m.ck, f[gz, gy, gx] * h)
    assert np.array_equal(hex_mdf_model(ng, E=2.0, h=h).ck, np.full(f.size, 2.0 * h))
    blk = HexBlock(ng, (0, 0, 0), ng, h=h)
    grp, _, _ = hex_type_group(blk, f)
    assert np.array_equal(grp.ck, m.ck)
    for bad in (f[:, :, :-1], f.astype(np.float32), list(f.ravel())):
        with pytest.raises(ValueError):
            hex_mdf_model(ng, h=h, E_field=bad)


def test_field_operators_match_element_assembly():
    """The host EBE operator of hex_type_group(E_field) (partition.TypeGroup arithmetic) equals the voxel_cases assembly,
    boxes with and without the clamped face."""
    from pcg_mpi_solver_b200.hexmesh import HexBlock, block_field, hex_type_group
    ng = (8, 6, 4)
    f = V.random_field(ng, seed=4)
    for e0, ne in (((0, 0, 0), (4, 6, 4)), ((4, 0, 0), (4, 6, 4)), ((2, 2, 1), (5, 3, 2))):
        blk = HexBlock(ng, e0, ne, h=0.5)
        fb = block_field(f, blk)
        grp, eff, ndof = hex_type_group(blk, fb)
        A = V.assemble(V.fine_elements(fb, 0.5, grp.ke), ng, e0)
        x = np.random.default_rng(1).standard_normal(A.shape[0])
        xf = np.zeros(ndof)
        xf[eff] = x
        y = np.zeros(ndof)
        np.add.at(y, grp.loc_dof, grp.ke @ (grp.ck * xf[grp.loc_dof]))
        assert np.all(np.abs(y[eff] - A @ x) <= 1e-13 * (abs(A) @ np.abs(x))), e0


# host MG-PCG (Galerkin levels) and host Jacobi-PCG iterations to 1e-8 on the 16^3 two-phase box (inclusion_field, seed 3,
# fraction 0.4, radii 1..3) by contrast; measured with this restatement, recorded in DESIGN.md section 2.5
HOST_ITERS = {1: (11, 145), 10: (18, 362), 100: (47, 611), 1000: (122, 1074)}


@pytest.mark.parametrize("contrast", sorted(HOST_ITERS))
def test_host_mg_pcg_converges_across_contrast(contrast):
    ne, h = (16, 16, 16), 1.0 / 16
    f = V.two_phase(ne, contrast, seed=3)
    H = V.HostFieldMultigrid(f, h)
    b = G.load_vector(ne, h)
    x, itm = G.pcg(H.A[0], b, H.apply, 1e-8, 400)
    _, itj = G.pcg(H.A[0], b, lambda r: H.dinv[0] * r, 1e-8, 4000)
    assert np.linalg.norm(b - H.A[0] @ x) <= 1e-8 * np.linalg.norm(b)
    mg_ref, jac_ref = HOST_ITERS[contrast]
    assert abs(itm - mg_ref) <= 2 and abs(itj - jac_ref) <= 5, (itm, itj)
    assert itm < itj / 8


def test_field_entries_long_double_equal_the_assembly():
    """voxel_cases.field_entries_ld (the 256^3 reference, entry by entry) against assemble_ld on a small box: the same values,
    sums of |terms| and term counts."""
    from pcg_mpi_solver_b200.hexmesh import hex_element_stiffness
    f = V.random_field((5, 4, 3), seed=6)
    ke = hex_element_stiffness()
    rows, cols, val, mag, k = V.assemble_ld(V.fine_elements(f, 0.5, ke))
    v2, m2, k2 = V.field_entries_ld(f, 0.5, ke, rows, cols)
    assert np.array_equal(k, k2)
    # assemble_ld rounds each product Ck_e Ke to double first, field_entries_ld forms it in long double
    assert np.all(np.abs(val - v2) <= 2.0 ** -52 * mag) and np.all(np.abs(mag - m2) <= 2.0 ** -52 * mag)
