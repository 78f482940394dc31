"""Multi-rank worker for the index-free multigrid hierarchy across ranks (launched by tests/test_gpu_gmg_index_free_dd.py
through torch.distributed.run; argv: out.json pgrid per kind, kind csr or hexop, the fine operator).

Every rank builds its box of partition_blocks(ng, pgrid) (per^3 elements), its fine operator, HexMultigrid(op, block,
blocks=..., coarse="index_free"), and on its own the one-rank index-free hierarchy of the global mesh.  Checks, per rank:
- every smoothed ranked level's local product (level_apply) bit-identical to HexBoxOperator of the rank's box halved l
  times at spacing 2^l h;
- lambda within 1e-13 of the one-rank index-free lambda of the global mesh;
- the V-cycle within 1e-11 of gmg_cases.HostMultigrid(ng) fed the device's lambda;
- MG-PCG: flag 0 in the one-rank iteration count of the global mesh, x within 1e-9 of oracle ref_pcg (rank 0).
Ranks never raise on a mismatch: they record it, and rank 0 writes every rank's findings."""
import datetime
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

VCYCLE_TOL = 1e-11
LAMBDA_TOL = 1e-13


def main():
    out_path, pgrid, per, kind = sys.argv[1], tuple(int(v) for v in sys.argv[2].split(",")), int(sys.argv[3]), sys.argv[4]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    dist.init_process_group("gloo", timeout=datetime.timedelta(seconds=300))
    from oracle import ref_pcg as R
    from pcg_mpi_solver_b200.hexmesh import (HexBlock, generate_box_operator, generate_matrix, interface_lists, load_vector,
                                             partition_blocks)
    from pcg_mpi_solver_b200.hexop import HexBoxOperator
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator.from_torch_distributed(dev, nccl=False)
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

    def operator(b):
        return generate_matrix(b, device=dev) if kind == "csr" else generate_box_operator(b, device=dev)

    ng = tuple(pgrid[a] * per for a in range(3))
    h = 1.0 / ng[0]
    blocks = [HexBlock(b.ng, b.e0, b.ne, h=h) for b in partition_blocks(ng, pgrid)]
    blk = blocks[rank]
    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * G.nfree(ng)
    op = SubdomainOperator(operator(blk), comm, nbr, lists, w, n_global=n_global)
    mg = HexMultigrid(op, blk, blocks=blocks, coarse="index_free")
    info = mg.info()
    la = info["gather_level"]
    note(info["coarse"] == "index_free", "info() does not report an index-free hierarchy")
    gblk = HexBlock(ng, (0, 0, 0), ng, h=h)
    op1 = SubdomainOperator(generate_box_operator(gblk, device=dev))
    mg1 = HexMultigrid(op1, gblk, coarse="index_free")
    info1 = mg1.info()

    # the ranked levels' local products against the index-free operator of the rank's halved box
    rng = np.random.default_rng(100 + rank)
    lb = blk
    stats["ranked_levels_checked"] = 0
    for l in range(1, la):
        lb = HexBlock(tuple(v // 2 for v in lb.ng), tuple(v // 2 for v in lb.e0), tuple(v // 2 for v in lb.ne), h=2 * lb.h)
        x = t(rng.standard_normal(info["n"][l]))
        ref = HexBoxOperator(lb, device=dev).apply_local(x)
        note(torch.equal(mg.level_apply(l, x), ref), f"level {l} product not bit-identical to its box operator")
        stats["ranked_levels_checked"] += 1

    glam = info["global_lambda"]
    lam_err = max(abs(a - b) / b for a, b in zip(glam, info1["lambda"][:-1]))
    stats["lambda_rel_err"] = lam_err
    note(lam_err <= LAMBDA_TOL, f"lambda off the one-rank index-free lambda by {lam_err:.3e}")

    def gmap(b):
        lz, ly, lx = np.meshgrid(np.arange(b.ne[2] + 1), np.arange(b.ne[1] + 1), np.arange(b.x_lo, b.ne[0] + 1), indexing="ij")
        gn = ((lz.ravel() + b.e0[2]) * (b.ng[1] + 1) + ly.ravel() + b.e0[1]) * b.ng[0] + (lx.ravel() + b.e0[0] - 1)
        return (3 * gn[:, None] + np.arange(3)[None, :]).ravel()

    m0 = gmap(blk)
    host = G.HostMultigrid(ng, h, lambdas=glam)
    r = np.random.default_rng(1234).standard_normal(n_global)          # the same draws on every rank
    z = mg.apply(t(r[m0])).cpu().numpy()
    want = host.apply(r)[m0]
    err = float(np.linalg.norm(z - want) / np.linalg.norm(want))
    stats["vcycle_rel_err"] = err
    note(err <= VCYCLE_TOL, f"V-cycle off the host by {err:.3e}")

    b = load_vector(blk, device=dev)
    x, si = op.solve(b, mg, 1e-8, 100)
    bg = load_vector(gblk, device=dev)
    _, s1 = op1.solve(bg, mg1, 1e-8, 100)
    stats["iters"], stats["iters_one_rank"] = si.iters, s1.iters
    note(si.flag == 0 and si.iters == s1.iters, f"flag {si.flag} iters {si.iters} vs one-rank {s1.iters}")

    xs = allg((m0, x.cpu().numpy(), fails, stats, time.time() - t0))
    if rank == 0:
        res = {"world": world, "pgrid": list(pgrid), "per": per, "kind": kind, "fails": [f for g in xs for f in g[2]],
               "stats": [g[3] for g in xs], "seconds": max(g[4] for g in xs)}
        xg = np.zeros(n_global)
        for m, v, *_ in xs:
            xg[m] = v
        A = R.hex_box_csr(ng, (0, 0, 0), ng, h=h)
        ref = R.ref_pcg([R.CsrPart(A, bg.cpu().numpy())], [1.0 / A.diagonal()], 1e-11, 20000)
        res["x_vs_ref"] = float(np.linalg.norm(xg - ref["X"][0]) / np.linalg.norm(ref["X"][0]))
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
