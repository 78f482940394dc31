"""Multi-rank worker for the multigrid preconditioner across ranks (launched by tests/test_gpu_gmg_dd.py through
torch.distributed.run; argv: out.json pgrid per kind).

Every rank builds its box of partition_blocks(ng, pgrid) (per^3 elements), its operator (csr / ebe_ordered / ebe) with the
interface lists of hexmesh, and HexMultigrid(op, block, blocks=...).  It also builds the one-rank HexMultigrid of the global
mesh on its own, as the reference of the parts.  Checks, per rank:
- lambda and the level sizes bit-identical on every rank, lambda within 1e-10 of the one-rank lambda of the global mesh;
- prolongation bit-identical to the one-rank device prolongation of the global vector, on every ranked level;
- restriction (with the coarse exchange-add) within (27 + 8 + 2) 2^-53 sum|terms| of the host P^T r;
- the gathered vector equal to the global vector bit for bit, and it and the coarse solve bit-identical on every rank;
- the whole V-cycle against gmg_cases.HostMultigrid(ng, lambdas=device lambda) (bound VCYCLE_TOL, the maximum is reported),
  shared-dof copies of z agreeing across ranks, two V-cycles of one input bit-identical (not on the atomic EBE operator);
- MG-PCG: flag 0 within +-1 iteration of the one-rank MG-PCG of the global mesh, x within 1e-9 of oracle ref_pcg (rank 0),
  graph on/off x check_every 1/7 bit-identical x and traces, traces identical across ranks but for rank / local and
  replayed by tests/pcg_shadow.py, flag 1 at maxiter, flag 2 on every rank from a NaN in rank 0's Minv;
- refusals (host side and the C entry point) that allocate nothing.
Ranks never raise on a mismatch: they record it, and rank 0 writes every rank's findings."""
import datetime
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist

from tests import gmg_cases as G

EPS = 2.0 ** -53
VCYCLE_TOL = 1e-11      # ||z - z_host|| / ||z_host||: distributed sums round differently from the one-rank order


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    out_path, pgrid, per, kind = sys.argv[1], tuple(int(v) for v in sys.argv[2].split(",")), int(sys.argv[3]), sys.argv[4]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    timeout = datetime.timedelta(seconds=300)
    if shared:
        dist.init_process_group("gloo", timeout=timeout)
    else:
        dist.init_process_group("nccl", device_id=dev, timeout=timeout)
    from oracle import ref_pcg as R
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix, interface_lists, load_vector, partition_blocks
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    from tests.mgpu_worker import trace_checks
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    transport = comm.transport
    fails, stats = [], {}
    t0 = time.time()

    def allg(obj):
        box = [None] * world
        dist.all_gather_object(box, obj)
        return box

    def t(v):
        return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)

    def note(ok, what):
        if not ok:
            fails.append(f"rank {rank} {what}")

    ng = tuple(pgrid[a] * per for a in range(3))
    h = 1.0 / ng[0]
    blocks = [HexBlock(b.ng, b.e0, b.ne, h=h) for b in partition_blocks(ng, pgrid)]
    blk = blocks[rank]

    def operator(b):
        return generate_matrix(b, device=dev) if kind == "csr" else generate_ebe(b, device=dev, ordered=kind == "ebe_ordered")

    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * G.nfree(ng)
    op = SubdomainOperator(operator(blk), comm, nbr, lists, w, n_global=n_global)
    mg = HexMultigrid(op, blk, blocks=blocks)
    info = mg.info()
    la = info["gather_level"]
    # the one-rank hierarchy of the global mesh, built by every rank on its own
    gblk = HexBlock(ng, (0, 0, 0), ng, h=h)
    op1 = SubdomainOperator(operator(gblk))
    mg1 = HexMultigrid(op1, gblk)
    info1 = mg1.info()
    allinfo = allg((info["n"][la + 1:], [float(v).hex() for v in info["lambda"]], info["levels"]))
    note(all(a[1:] == allinfo[0][1:] and a[0] == allinfo[0][0] for a in allinfo), "lambda / level sizes differ across ranks")
    glam = info["global_lambda"]
    note(info["levels"] - 1 == info1["levels"], f"levels {info['levels']} vs one-rank {info1['levels']}")
    lam_err = max(abs(a - b) / b for a, b in zip(glam, info1["lambda"][:-1]))
    stats["lambda_rel_err"] = lam_err
    note(lam_err <= 1e-10, f"lambda off the one-rank lambda by {lam_err:.3e}")
    note(glam[la:] == info1["lambda"][la:], "replicated levels' lambda differ from the one-rank ones")

    # per-level boxes and global dof maps (hexmesh numbering, global box x = 0 clamped)
    def half(b):
        return HexBlock(tuple(v // 2 for v in b.ng), tuple(v // 2 for v in b.e0), tuple(v // 2 for v in b.ne), h=2 * b.h)

    lvl = [blocks]
    for _ in range(la):
        lvl.append([half(b) for b in lvl[-1]])

    def gmap(b):
        lz, ly, lx = np.meshgrid(np.arange(b.ne[2] + 1), np.arange(b.ne[1] + 1), np.arange(b.x_lo, b.ne[0] + 1), indexing="ij")
        gn = ((lz.ravel() + b.e0[2]) * (b.ng[1] + 1) + ly.ravel() + b.e0[1]) * b.ng[0] + (lx.ravel() + b.e0[0] - 1)
        return (3 * gn[:, None] + np.arange(3)[None, :]).ravel()

    maps = [gmap(lv[rank]) for lv in lvl]
    rng = np.random.default_rng(1234)            # the same draws on every rank
    for l in range(la):
        ngf, ngc = lvl[l][0].ng, lvl[l + 1][0].ng
        ec, xf = rng.standard_normal(3 * G.nfree(ngc)), rng.standard_normal(3 * G.nfree(ngf))
        got = mg.prolong_add(l, t(ec[maps[l + 1]]), t(xf[maps[l]])).cpu().numpy()
        want = mg1.prolong_add(l, t(ec), t(xf)).cpu().numpy()[maps[l]]
        note(np.array_equal(got.view(np.uint64), want.view(np.uint64)), f"prolongation level {l} not bit-identical")
        rf = rng.standard_normal(3 * G.nfree(ngf))
        got = mg.restrict(l, t(rf[maps[l]])).cpu().numpy()
        ref, mag = G.restrict(rf, ngf, np.longdouble)
        ok = np.abs(got - ref[maps[l + 1]].astype(np.float64)) <= (27 + 8 + 2) * EPS * mag[maps[l + 1]].astype(np.float64)
        note(bool(np.all(ok)), f"restriction level {l}: {int(np.sum(~ok))} entries off")
    vg = rng.standard_normal(info["n_gathered"])
    gathered = mg.gather(t(vg[maps[la]])).cpu().numpy()
    note(np.array_equal(gathered.view(np.uint64), vg.view(np.uint64)), "gathered vector differs from the global one")
    zc = mg.coarse_solve(t(rng.standard_normal(info["n"][-1]))).cpu().numpy()
    back = mg.scatter(t(vg)).cpu().numpy()
    note(np.array_equal(back, vg[maps[la]]), "scatter")
    shas = allg((_sha(gathered), _sha(zc)))
    note(all(s == shas[0] for s in shas), "gathered vector / coarse solve differ across ranks")

    # the whole V-cycle
    host = G.HostMultigrid(ng, h, lambdas=glam)
    r = rng.standard_normal(n_global)
    zt = mg.apply(t(r[maps[0]]))
    z = zt.cpu().numpy()
    want = host.apply(r)
    err = np.linalg.norm(z - want[maps[0]]) / np.linalg.norm(want[maps[0]])
    stats["vcycle_rel_err"] = err
    note(err <= VCYCLE_TOL, f"V-cycle off the host by {err:.3e}")
    if kind != "ebe":
        z2 = mg.apply(t(r[maps[0]]))
        note(torch.equal(zt, z2), "two V-cycles of one input differ")
    allz = allg((maps[0], z))
    zg = np.full(n_global, np.nan)
    spread = 0.0
    for m, v in allz:
        seen = ~np.isnan(zg[m])
        spread = max(spread, float(np.max(np.abs(zg[m][seen] - v[seen]), initial=0.0)))
        zg[m] = v
    stats["z_copy_spread"] = spread / np.abs(want).max()
    note(spread <= 1e-13 * np.abs(want).max(), f"shared copies of z differ by {spread:.3e}")

    # MG-PCG across ranks
    b = load_vector(blk, device=dev)
    x, si = op.solve(b, mg, 1e-8, 100)
    bg = load_vector(gblk, device=dev)
    _, s1 = op1.solve(bg, mg1, 1e-8, 100)
    stats["iters"], stats["iters_one_rank"] = si.iters, s1.iters
    note(si.flag == 0 and abs(si.iters - s1.iters) <= 1, f"flag {si.flag} iters {si.iters} vs one-rank {s1.iters}")
    base, i0 = op.solve(b, mg, 1e-12, 200, trace=True, check_every=1, use_graph=False)
    stats["flag_1e-12"] = i0.flag
    note(i0.flag in (0, 3), f"tol 1e-12 flag {i0.flag}")    # long boxes (24 x 8 x 8) stagnate just above 1e-12
    if kind != "ebe":
        for use_graph in (False, True):
            for check_every in (1, 7):
                xx, ii = op.solve(b, mg, 1e-12, 200, trace=True, check_every=check_every, use_graph=use_graph)
                note(torch.equal(xx, base) and ii.trace.tobytes() == i0.trace.tobytes(), f"graph {use_graph} check_every {check_every}")
    _, im = op.solve(b, mg, 1e-14, 3)
    note(im.flag == 1 and im.iters <= 3, f"maxiter: flag {im.flag}")
    minv = op.jacobi()
    if rank == 0:
        minv[5] = float("nan")
    bad = HexMultigrid(op, blk, minv=minv, blocks=blocks)
    _, ib = op.solve(b, bad, 1e-8, 50)
    note(ib.flag == 2, f"NaN in rank 0's Minv: flag {ib.flag}")
    del bad

    # refusals: nothing allocated
    lib = _lib.load()
    import ctypes
    import gc
    gc.collect()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    refusals = 0
    for what, kw in (("block not blocks[rank]", dict(blocks=blocks[1:] + blocks[:1])),
                     ("no blocks", dict(blocks=None)),
                     ("gap", dict(blocks=[HexBlock(ng, (0, 0, 0), (2, 2, 2), h=h) if k != rank else blk for k in range(world)]))):
        try:
            HexMultigrid(op, blk, **kw)
            fails.append(f"rank {rank} refusal {what}: accepted")
        except ValueError:
            refusals += 1
    box = blk.cbox()
    halos = (ctypes.c_void_p * (la + 8))(*([hh.value for hh in mg._halos[:la]] + [None] * 8))
    owns = (ctypes.c_void_p * (la + 9))()
    out = ctypes.c_void_p()
    ke = np.ascontiguousarray(np.eye(24))
    rc = lib.pcgb_mg_create_ranks(op._solver, ctypes.byref(box), la + 8, halos, mg._gather, owns,
                                  ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 1.0, h, _lib.ptr(minv), 2, 0.25, ctypes.byref(out))
    note(rc == -1 and not out, f"pcgb_mg_create_ranks with too many levels: rc {rc}")
    refusals += rc == -1
    torch.cuda.synchronize()
    note(torch.cuda.mem_get_info(dev)[0] >= free0, "a refusal allocated device memory")
    stats["refusals"] = refusals

    torch.cuda.synchronize()
    status = lib.pcgb_comm_status(comm.handle, _lib.stream_ptr())
    note(status == 0, f"communicator status {status}")
    xs = allg((maps[0], base.cpu().numpy(), {"trace": i0.trace, "trace_total": i0.trace_total}, fails, stats, time.time() - t0))
    if rank == 0:
        res = {"world": world, "pgrid": list(pgrid), "per": per, "kind": kind, "transport": transport,
               "fails": [f for g in xs for f in g[3]], "stats": [g[4] for g in xs], "seconds": max(g[5] for g in xs)}
        res.update(trace_checks([g[2] for g in xs], transport, 1e-12, 200, n_global))
        xg = np.zeros(n_global)
        for m, v, *_ in xs:
            xg[m] = v
        A = R.hex_box_csr(ng, (0, 0, 0), ng, h=h)
        bh = bg.cpu().numpy()
        ref = R.ref_pcg([R.CsrPart(A, bh)], [1.0 / A.diagonal()], 1e-11, 20000)
        res["x_vs_ref"] = float(np.linalg.norm(xg - ref["X"][0]) / np.linalg.norm(ref["X"][0]))
        res["ref_flag"] = int(ref["Flag"])
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
