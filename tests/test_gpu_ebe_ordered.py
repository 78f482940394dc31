"""The ordered matrix-free operator (csrc/ebe_ordered.cuh, EbeMatrixOrdered): entrywise against a long-double
restatement at every kernel edge, its summation order pinned bit for bit, bit-reproducible applications and solves,
parity with the oracle inside PCG, and argument refusals that leak nothing."""
import dataclasses
import gc
import json
import os

import numpy as np
import pytest

from oracle import ref_pcg as R
from tests import asm_cases as AC
from tests import ebe_ordered_cases as C
from tests import pcg_shadow as S
from tests.test_gpu_ebe import SIGNS, _bench_boxes, _spd_groups, _synthetic_groups

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _apply(E, x, cuda):
    """E applied to x into a NaN-filled output (every entry must be written)."""
    import torch
    y = torch.full((E.shape[0],), float("nan"), dtype=torch.float64, device=cuda)
    E.apply_local(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to(cuda), out=y)
    return y.cpu().numpy()


def _ordered(groups, eff, ndof, cuda):
    from pcg_mpi_solver_b200.ebe import EbeMatrixOrdered
    return EbeMatrixOrdered(groups, eff, ndof, device=cuda)


@pytest.mark.parametrize("signs", list(SIGNS))
def test_synthetic_groups_entrywise(cuda, signs):
    """Pattern sizes 1..96 around the thread kernel (24) and the lane passes (32 / 64 / 96), block tails, no / some / all
    sign flips, clamped dofs, a fully clamped element, high-valence and untouched free dofs - entrywise, through
    apply_local and through the solver's pcgb_apply."""
    import torch
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    rng = np.random.default_rng(100 + list(SIGNS).index(signs))
    groups, eff, ndof = _synthetic_groups(rng, SIGNS[signs])
    gc.collect()
    E = _ordered(groups, eff, ndof, cuda)
    x = rng.standard_normal(len(eff))
    C.assert_entrywise(_apply(E, x, cuda), groups, eff, ndof, x)
    op = SubdomainOperator(E)
    y = torch.full((len(eff),), float("nan"), dtype=torch.float64, device=cuda)
    op.apply(torch.from_numpy(x).to(cuda), out=y)
    C.assert_entrywise(y.cpu().numpy(), groups, eff, ndof, x)


def _asm_subs():
    subs = [(f"pattern-{nd}-{v}", AC.pattern_case(nd, v)) for nd in AC.PATTERN_SIZES if nd <= 96 for v in AC.PATTERN_VARIANTS]
    subs += [("structure", AC.structure_case()), ("no_rows", AC.no_rows_case()), ("many_groups", AC.many_groups_case()),
             ("duplicate", AC.duplicate_case()), ("order", AC.order_case()), ("spd", AC.spd_case())]
    return subs


def test_asm_cases_entrywise(cuda):
    """The assembly's edge cases with nd <= 96 (non-symmetric Ke, a dof shared by 200 elements, free dofs no element
    touches, n = 0, 300 groups, an element listing one free dof twice) against the long-double restatement."""
    rng = np.random.default_rng(3)
    for name, sub in _asm_subs():
        E = _ordered(sub.groups, sub.loc_dof_eff, sub.ndof, cuda)
        x = rng.standard_normal(sub.n)
        y = _apply(E, x, cuda)
        assert y.shape == (sub.n,), name
        C.assert_entrywise(y, sub.groups, sub.loc_dof_eff, sub.ndof, x)
        if name == "structure":
            pos = np.searchsorted(sub.loc_dof_eff, sub.extra["empty"])
            assert (y[pos] == 0.0).all()


def test_tiny_operators(cuda):
    """n = 0 and n = 1 (one element, one free dof, pattern sizes 1 and 24)."""
    from pcg_mpi_solver_b200.partition import TypeGroup
    E = _ordered([TypeGroup(0, np.zeros((3, 2), np.int64), np.zeros((3, 2), bool), np.ones(2), np.eye(3), np.arange(2))],
                 np.zeros(0, np.int64), 1, cuda)
    assert _apply(E, np.zeros(0), cuda).shape == (0,)
    for nd in (1, 24):
        ke = np.arange(1.0, nd * nd + 1).reshape(nd, nd)
        g = TypeGroup(0, np.arange(nd)[:, None], np.zeros((nd, 1), bool), np.array([0.5]), ke, np.arange(1))
        E = _ordered([g], np.array([0]), nd, cuda)
        assert _apply(E, np.array([3.0]), cuda)[0] == 0.5 * 3.0 * ke[0, 0]


def test_order_pin(cuda):
    """Phase-1 products exact (integer data), per-dof sums that cancel: y is bit-equal to the documented (group, local
    index, element) order, which differs from the (group, element, local index) order."""
    groups, eff, ndof, x, want = C.order_pin()
    y = _apply(_ordered(groups, eff, ndof, cuda), x, cuda)
    assert np.array_equal(y, want), y
    assert not np.array_equal(y, C.ordered_f64(groups, eff, ndof, x, order="element"))


def test_small_cases_bit_equal_to_documented_order(cuda):
    """On small cases with general data, both phases as documented in fp64 (exact fma) give y bit for bit."""
    rng = np.random.default_rng(8)
    for sub in (AC.duplicate_case(), AC.structure_case(), AC.pattern_case(33, "signs20"), AC.pattern_case(24, "signsall")):
        x = rng.standard_normal(sub.n)
        y = _apply(_ordered(sub.groups, sub.loc_dof_eff, sub.ndof, cuda), x, cuda)
        assert np.array_equal(y, C.ordered_f64(sub.groups, sub.loc_dof_eff, sub.ndof, x))


def test_hex_24dof_constant_and_generic_paths_and_two_live_operators(cuda):
    """The 24-dof pattern on the constant-memory kernel and, once the slot table is full, on the warp kernel: bit-equal
    results; two live operators with different Ke keep their own matrices."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_type_group
    blk = HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4), h=0.25, nu=0.3)
    grp, eff, ndof = hex_type_group(blk)
    x = np.random.default_rng(4).standard_normal(len(eff))
    E1 = _ordered([grp], eff, ndof, cuda)
    y1 = _apply(E1, x, cuda)
    C.assert_entrywise(y1, [grp], eff, ndof, x)
    # fill the constant-memory table with other 24-dof patterns, then the same group goes to the warp kernel
    rng = np.random.default_rng(5)
    fillers = []
    for _ in range(8):
        ke = rng.standard_normal((24, 24))
        fillers.append(_ordered([dataclasses.replace(grp, ke=ke + ke.T)], eff, ndof, cuda))
    blk2 = HexBlock((6, 5, 4), (0, 0, 0), (6, 5, 4), h=0.25, nu=0.45)
    grp2, _, _ = hex_type_group(blk2)
    E2 = _ordered([grp2], eff, ndof, cuda)                  # no free slot: warp kernel
    y2 = _apply(E2, x, cuda)
    C.assert_entrywise(y2, [grp2], eff, ndof, x)
    assert np.array_equal(_apply(E1, x, cuda), y1)          # the first operator still has its own matrix
    del fillers
    gc.collect()
    E1w = _ordered([grp], eff, ndof, cuda)                   # E1 still holds its slot: the same Ke shares it by content
    assert np.array_equal(_apply(E1w, x, cuda), y1)
    del E1, E1w
    gc.collect()
    fillers = [_ordered([dataclasses.replace(grp, ke=(lambda k: k + k.T)(rng.standard_normal((24, 24))))], eff, ndof, cuda)
               for _ in range(8)]
    E1g = _ordered([grp], eff, ndof, cuda)                   # same pattern on the warp kernel: same bits
    assert np.array_equal(_apply(E1g, x, cuda), y1)
    del fillers
    gc.collect()
    torch.cuda.synchronize()


def test_reproducible_applications_and_instances(cuda):
    rng = np.random.default_rng(9)
    groups, eff, ndof = _synthetic_groups(rng, 0.2)
    gc.collect()
    x = rng.standard_normal(len(eff))
    E1, E2 = _ordered(groups, eff, ndof, cuda), _ordered(groups, eff, ndof, cuda)
    y = _apply(E1, x, cuda)
    assert np.array_equal(_apply(E1, x, cuda), y) and np.array_equal(_apply(E2, x, cuda), y)


def _case(kind, cuda, rng):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    if kind == "synthetic":
        groups, eff, ndof, A = _spd_groups(rng)
        E = _ordered(groups, eff, ndof, cuda)
    else:
        blk = HexBlock((8, 6, 5), (0, 0, 0), (8, 6, 5), h=1.0 / 8)
        E, A = generate_ebe(blk, device=cuda, ordered=True), R.hex_box_csr(blk.ng, blk.e0, blk.ne, h=blk.h)
    return SubdomainOperator(E), A, rng.standard_normal(A.shape[0])


def test_solve_bit_reproducible_across_batching(cuda):
    """x and resvec bit-identical over two runs, graph capture on and off, and check_every 1, 7 and 16."""
    import torch
    op, A, b = _case("synthetic", cuda, np.random.default_rng(7))
    bd = torch.from_numpy(b).to(cuda)
    minv = op.jacobi()
    base, info0 = op.solve(bd, minv, 1e-10, 1000, record_resvec=True, check_every=1, use_graph=False)
    assert info0.flag == 0
    for use_graph in (False, True):
        for check_every in (1, 7, 16):
            for _ in range(2):
                x, info = op.solve(bd, minv, 1e-10, 1000, record_resvec=True, check_every=check_every, use_graph=use_graph)
                assert torch.equal(x, base), (use_graph, check_every)
                assert np.array_equal(info.resvec, info0.resvec) and info.iters == info0.iters and info.relres == info0.relres


@pytest.mark.parametrize("kind", ["synthetic", "hex"])
def test_solver_matches_oracle(cuda, kind):
    from pcg_mpi_solver_b200 import solve
    op, A, b = _case(kind, cuda, np.random.default_rng(5))
    minv = 1.0 / A.diagonal()
    resvec = []
    ref = R.ref_pcg([R.CsrPart(A, b)], [minv], 1e-13, 5000, resvec=resvec)
    x, flag, relres, iters, info = solve(op, b, "jacobi", 1e-13, 5000, return_info=True, record_resvec=True)
    assert flag == ref["Flag"] == 0 and abs(iters - ref["Iter"]) <= 2
    assert np.linalg.norm(x - ref["X"][0]) <= 1e-10 * np.linalg.norm(ref["X"][0])
    k = min(12, len(resvec), len(info.resvec))
    np.testing.assert_allclose(info.resvec[:k], np.asarray(resvec[:k]), rtol=1e-9)


def test_solver_matches_oracle_partitioned_hex(cuda, tmp_path):
    """The mdf pipeline (partition_mesh -> to_operator(kind="ebe_ordered")) against the assembled matrix and the oracle."""
    import torch
    from oracle.hex_mdf import write_hex_mdf
    from pcg_mpi_solver_b200.model import load_mdf
    from pcg_mpi_solver_b200.partition import partition_mesh
    write_hex_mdf(str(tmp_path), (9, 7, 5))
    sub = partition_mesh(load_mdf(str(tmp_path)), 1, assemble=True)[0]
    op = sub.to_operator(device=cuda, kind="ebe_ordered")
    x = np.random.default_rng(0).standard_normal(sub.n)
    y = op.apply(torch.from_numpy(x).to(cuda)).cpu().numpy()
    assert np.abs(y - sub.A @ x).max() <= 1e-12 * (abs(sub.A) @ np.abs(x)).max()
    np.testing.assert_allclose(op.jacobi().cpu().numpy(), 1.0 / sub.A.diagonal(), rtol=1e-13)
    xs, info = op.solve(torch.from_numpy(sub.b).to(cuda), op.jacobi(), 1e-10, 5000)
    ref = R.ref_pcg([R.CsrPart(sub.A, sub.b)], [1.0 / sub.A.diagonal()], 1e-10, 5000)
    assert info.flag == ref["Flag"] == 0 and abs(info.iters - ref["Iter"]) <= 2


def test_trace_replays(cuda):
    """A traced solve replays through the host restatement of the control logic bit for bit."""
    import torch
    op, A, b = _case("hex", cuda, np.random.default_rng(12))
    x, info = op.solve(torch.from_numpy(b).to(cuda), op.jacobi(), 1e-12, 3000, trace=True, check_every=8)
    assert info.flag == 0 and info.trace_total == len(info.trace) > 0
    sh = S.replay(info.trace, 1e-12, 3000, A.shape[0])
    assert sh.result["flag"] == info.flag


def test_agrees_with_ebe_and_csr_on_bench_boxes(cuda):
    """On every box the bench uses: the ordered operator within the entrywise bound, and against EbeMatrix and the
    generated CSR matrix within 1e-13 of sum |A||x|."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import generate_ebe, generate_matrix, hex_type_group
    rng = np.random.default_rng(13)
    for blk in _bench_boxes():
        grp, eff, ndof = hex_type_group(blk)
        O, E, A = generate_ebe(blk, device=cuda, ordered=True), generate_ebe(blk, device=cuda), generate_matrix(blk, device=cuda)
        x = rng.standard_normal(blk.n)
        xd = torch.from_numpy(x).to(cuda)
        yo = _apply(O, x, cuda)
        C.assert_entrywise(yo, [grp], eff, ndof, x)
        bound = abs(A.to_scipy()) @ np.abs(x)
        for other in (E.apply_local(xd).cpu().numpy(), A.spmv(xd).cpu().numpy()):
            assert (np.abs(yo - other) <= 1e-13 * bound).all(), (blk.e0, blk.ne)


def test_concrete(cuda):
    import torch
    from pcg_mpi_solver_b200.partition import partition_mesh
    zp = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "concrete.zip")
    if not os.path.exists(zp):
        pytest.skip("concrete.zip not staged")
    sub = partition_mesh(zp, 1, assemble=False)[0]
    op = sub.to_operator(device=cuda, kind="ebe_ordered")
    csr = sub.to_operator(device=cuda, kind="csr")
    x = torch.randn(sub.n, dtype=torch.float64, device=cuda)
    yo, yc = op.apply(x), csr.apply(x)
    assert float((yo - yc).abs().max() / yc.abs().max()) <= 1e-12
    xs, info = op.solve(torch.from_numpy(sub.b).to(cuda), op.jacobi(), 1e-7, 10000)
    assert info.flag == 0 and abs(info.iters - 1085) <= 2


def test_hex_256_sampled_rows(cuda):
    """The 256^3 box (about 4.0e8 element slots): sampled rows against a long-double recomputation."""
    import torch
    from pcg_mpi_solver_b200.ebe import EbeMatrixOrdered
    from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_type_group
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 24 * 2**30:
        pytest.skip(f"needs 24 GiB free device memory, {free / 2**30:.1f} GiB free")
    B = 256
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    grp, eff, ndof = hex_type_group(blk)
    assert grp.loc_dof.size > 4.0e8
    E = EbeMatrixOrdered([grp], eff, ndof, device=cuda)
    rng = np.random.default_rng(256)
    x = rng.standard_normal(len(eff))
    y = E.apply_local(torch.from_numpy(x).to(cuda)).cpu().numpy()
    assert not np.isnan(y).any()
    # rows: random ones plus the first and last free dofs; their elements from the structure of the box
    rows = np.unique(np.concatenate([rng.integers(0, len(eff), 3000), np.arange(6), len(eff) - 1 - np.arange(6)]))
    xf = np.zeros(ndof, dtype=np.longdouble)
    xf[eff] = x
    nx = ny = nz = B
    for r in rows:
        node, d = divmod(int(eff[r]), 3)
        lx, rest = node % (nx + 1), node // (nx + 1)
        ly, lz = rest % (ny + 1), rest // (ny + 1)
        acc, scale = np.longdouble(0), np.longdouble(0)
        for dz in (0, 1):
            for dy in (0, 1):
                for dx in (0, 1):
                    ex, ey, ez = lx - dx, ly - dy, lz - dz
                    if not (0 <= ex < nx and 0 <= ey < ny and 0 <= ez < nz):
                        continue
                    e = (ez * ny + ey) * nx + ex
                    a = 3 * (dx + 2 * dy + 4 * dz) + d
                    u = np.longdouble(grp.ck[e]) * xf[grp.loc_dof[:, e]]
                    ke = grp.ke[a].astype(np.longdouble)
                    acc += ke @ u
                    scale += np.abs(ke) @ np.abs(u)
        assert abs(np.longdouble(y[r]) - acc) <= (8 * 25 + 2) * C.EPS * scale, r


def test_argument_errors_leak_nothing(cuda):
    """Null arrays, nd > 96 and n >= 2^30 return PCGB_ERR_ARG and leave the device allocation where it was (20 refusals)."""
    import ctypes
    import torch
    from pcg_mpi_solver_b200 import _lib
    lib = _lib.load()
    idx = torch.zeros((24, 4), dtype=torch.int32, device=cuda)
    ck = torch.ones(4, dtype=torch.float64, device=cuda)
    ke = np.eye(97)

    def group(nd, with_idx=True, with_ck=True):
        g = (_lib.EbeGroup * 1)()
        g[0].nd, g[0].ne = nd, 4
        g[0].d_idx = idx.data_ptr() if with_idx else None
        g[0].d_ck = ck.data_ptr() if with_ck else None
        g[0].d_sign = None
        g[0].ke_host = ke.ctypes.data
        return g

    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(cuda)
    free0, _ = torch.cuda.mem_get_info(cuda)
    h = ctypes.c_void_p()
    for _ in range(4):
        for n, g in ((8, group(24, with_idx=False)), (8, group(24, with_ck=False)), (8, group(97)), (2**30, group(24)),
                     (8, None)):
            rc = lib.pcgb_ebe_ordered_create(n, 1, g, ctypes.byref(h))
            assert rc == -1 and not h, lib.pcgb_last_error()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(cuda) == before
    free1, _ = torch.cuda.mem_get_info(cuda)
    assert free1 >= free0
    assert lib.pcgb_solver_create_ebe_ordered(None, None, None, ctypes.byref(h)) == -1
    assert lib.pcgb_ebe_ordered_apply(None, None, None, None) == -1


def test_residual_history_128_matches_golden(cuda):
    """The bench's 128^3 box with the ordered operator against the oracle's committed residual history."""
    import torch
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 8 * 2**30:
        pytest.skip("needs 8 GiB free device memory")
    B = 128
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    op = SubdomainOperator(generate_ebe(blk, device=cuda, ordered=True))
    b = load_vector(blk, device=cuda)
    gold = json.load(open(os.path.join(HERE, "golden", f"hex{B}_N1_resvec.json")))
    x, info = op.solve(b, op.jacobi(), 0.0, 40, fixed_iters=True, record_resvec=True, check_every=20)
    ref = np.array(gold["resvec"])
    np.testing.assert_allclose(info.resvec[:11], ref[:11], rtol=1e-9)
    np.testing.assert_allclose(info.resvec[:41], ref[:41], rtol=1e-7)
    x2, info2 = op.solve(b, op.jacobi(), 0.0, 40, fixed_iters=True, record_resvec=True, check_every=20)
    assert torch.equal(x, x2) and np.array_equal(info.resvec, info2.resvec)


# ------------------------------------------------------------------------------------------------------------- multi-rank
def _run_worker(world, tmp_path, block, graph, port, env, timeout=900):
    import subprocess
    import sys
    out = tmp_path / f"ebo_{world}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "ebe_ordered_worker.py"), str(out), str(block), str(graph)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads(out.read_text())


def _check_multi(res):
    assert res["flag"] == res["ref_flag"] == 0 and abs(res["iters"] - res["ref_iters"]) <= 2
    assert res["relres"] <= 1e-12 and res["x_rel_err"] <= 1e-9 and res["y_rel_err"] <= 1e-13
    assert res["same_x_all_ranks"] and res["same_y_all_ranks"]
    assert all(tuple(i) == tuple(res["all_infos"][0]) for i in res["all_infos"])
    assert res["trace_records"] > 0 and res["trace_complete"] and res["trace_identical"]
    assert res["trace_replayed"] is True, res["trace_replayed"]
    if res["transport"] == "peer":
        assert res["trace_sum_checked"] > 0 and res["trace_sum_mismatches"] == 0


@pytest.mark.parametrize("world,graph,block", [(2, 1, 6), (2, 0, 6), (4, 1, 5)])
def test_ranks_sharing_one_gpu(cuda, tmp_path, world, graph, block):
    """2 and 4 ranks time-sharing cuda:0 over the peer transport, against the oracle's multi-part emulation."""
    res = _run_worker(world, tmp_path, block, graph, 29817 + 2 * world + graph,
                      {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"})
    assert res["transport"] == "peer"
    _check_multi(res)


@pytest.mark.parametrize("transport", ["peer", "nccl"])
def test_two_gpus(cuda, tmp_path, transport):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    res = _run_worker(2, tmp_path, 6, 1, 29867 + (1 if transport == "nccl" else 0),
                      {"PCGB_COMM": transport, "PCGB_EXPECT_TRANSPORT": transport})
    assert res["transport"] == transport
    _check_multi(res)
