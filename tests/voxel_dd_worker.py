"""Multi-rank worker for voxel models (launched by tests/test_gpu_voxel_dd.py through torch.distributed.run; argv: out.json
pgrid per contrast).

Every rank draws the same global inclusion_field, cuts its box out with block_field, generates its own field operator
(no communication beyond the solve's halo exchange and reductions) and runs Jacobi-PCG across ranks.  Each rank also solves
the whole mesh on its own with the same field, as the reference.  Checks, per rank:
- flag and iterations equal to the one-rank solve's (+-2), x within 1e-9 of the one-rank x on the rank's dofs;
- the diagonal of the rank's field operator after the interface sum equal to the one-rank diagonal on its dofs (1e-14);
- HexMultigrid(..., E_field=...) refused with ValueError on a multi-rank operator, allocating nothing.
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

TOL = 1e-10     # 1e-11 stagnates (flag 3) on the one-rank solve of the contrast-100 box as well


def main():
    out_path, pgrid, per, contrast = sys.argv[1], tuple(int(v) for v in sys.argv[2].split(",")), int(sys.argv[3]), float(sys.argv[4])
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
    from pcg_mpi_solver_b200.hexmesh import (HexBlock, block_field, generate_matrix, inclusion_field, interface_lists, load_vector,
                                             partition_blocks)
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    fails, stats = [], {}
    t0 = time.time()

    def note(ok, what):
        if not ok:
            fails.append(f"rank {rank} {what}")

    ng = tuple(pgrid[a] * per for a in range(3))
    h = 1.0 / ng[0]
    blocks = [HexBlock(b.ng, b.e0, b.ne, h=h) for b in partition_blocks(ng, pgrid)]
    blk = blocks[rank]
    field = inclusion_field(ng, 0.4, (1.0, per / 3), 1.0, contrast, seed=17)
    fb = block_field(field, blk)
    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    op = SubdomainOperator(generate_matrix(blk, device=dev, E_field=fb), comm, nbr, lists, w, n_global=n_global)
    b = load_vector(blk, device=dev)
    x, si = op.solve(b, op.jacobi(), TOL, 50000)

    # the whole mesh on this rank alone, the same field
    gblk = HexBlock(ng, (0, 0, 0), ng, h=h)
    op1 = SubdomainOperator(generate_matrix(gblk, device=dev, E_field=field))
    x1, s1 = op1.solve(load_vector(gblk, device=dev), op1.jacobi(), TOL, 50000)
    lz, ly, lx = np.meshgrid(np.arange(blk.ne[2] + 1), np.arange(blk.ne[1] + 1), np.arange(blk.x_lo, blk.ne[0] + 1), indexing="ij")
    gn = ((lz.ravel() + blk.e0[2]) * (ng[1] + 1) + ly.ravel() + blk.e0[1]) * ng[0] + (lx.ravel() + blk.e0[0] - 1)
    gmap = torch.from_numpy((3 * gn[:, None] + np.arange(3)[None, :]).ravel()).to(dev)
    ref = x1[gmap]
    err = float((x - ref).norm() / ref.norm())
    stats.update(flag=si.flag, iters=si.iters, flag_one_rank=s1.flag, iters_one_rank=s1.iters, x_vs_one_rank=err, e0=list(blk.e0))
    note(si.flag == s1.flag == 0 and abs(si.iters - s1.iters) <= 2, f"flag {si.flag} iters {si.iters} vs one rank {s1.flag} {s1.iters}")
    note(err <= 1e-9, f"x off the one-rank x by {err:.3e}")
    d = op.exchange_add(op.A.diagonal())
    d1 = op1.A.diagonal()[gmap]
    derr = float((d - d1).abs().max() / d1.abs().max())
    stats["diag_vs_one_rank"] = derr
    note(derr <= 1e-14, f"assembled diagonal off the one-rank one by {derr:.3e}")

    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    try:
        HexMultigrid(op, blk, E_field=fb, blocks=blocks)
        fails.append(f"rank {rank} HexMultigrid with E_field across ranks: accepted")
    except ValueError:
        stats["refused"] = True
    torch.cuda.synchronize()
    note(torch.cuda.mem_get_info(dev)[0] >= free0, "the refusal allocated device memory")

    box = [None] * world
    dist.all_gather_object(box, (fails, stats, time.time() - t0))
    if rank == 0:
        res = {"world": world, "pgrid": list(pgrid), "per": per, "contrast": contrast, "transport": comm.transport,
               "fails": [f for g in box for f in g[0]], "stats": [g[1] for g in box], "seconds": max(g[2] for g in box)}
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
