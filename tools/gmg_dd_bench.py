"""Jacobi-PCG against multigrid-preconditioned PCG across ranks on the bench's weak-scaled hex stacks (one box of
--block^3 elements per rank, hexmesh.block_grid / partition_blocks), one GPU per rank.

    torchrun --nproc-per-node 8 tools/gmg_dd_bench.py --block 128 --tol 1e-8 [--operator csr|ebe_ordered|ebe] [--coarse csr|index_free]

For each arm, per rank: iterations, flag, the device time of the loop (CUDA events inside the solve), the host wall time
of the whole solve (ending in a device synchronise and a barrier), and for the multigrid arm its set-up time and the
V-cycle time per application (CUDA events around `pcgb_mg_apply`).  Rank 0 prints one JSON line per arm with every
rank's numbers and the card's name, SM clock limit and power limit.  Ranks sharing one GPU (PCGB_SHARED_GPU=1) run, but
their times say nothing about speed.  --coarse index_free builds HexMultigrid(coarse="index_free"): index-free ranked and
replicated coarse levels.
"""
import argparse
import datetime
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.gmg_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", type=int, default=128)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--operator", choices=["csr", "ebe_ordered", "ebe"], default="csr")
    ap.add_argument("--degree", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--vcycles", type=int, default=20)
    ap.add_argument("--coarse", choices=["csr", "index_free"], default="csr")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        sys.exit("gmg_dd_bench: needs a CUDA device")
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    timeout = datetime.timedelta(seconds=600)
    if shared:
        dist.init_process_group("gloo", timeout=timeout)
    else:
        dist.init_process_group("nccl", device_id=dev, timeout=timeout)
    from pcg_mpi_solver_b200.hexmesh import HexBlock, block_grid, generate_ebe, generate_matrix, interface_lists, load_vector, partition_blocks
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    pgrid = block_grid(world)
    ng = tuple(pgrid[ax] * a.block for ax in range(3))
    blocks = [HexBlock(b.ng, b.e0, b.ne, h=1.0 / ng[0]) for b in partition_blocks(ng, pgrid)]
    blk = blocks[rank]
    A = generate_matrix(blk, device=dev) if a.operator == "csr" else generate_ebe(blk, device=dev, ordered=a.operator == "ebe_ordered")
    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    op = SubdomainOperator(A, comm, nbr, lists, w, n_global=n_global)
    b = load_vector(blk, device=dev)
    minv = op.jacobi()
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    mg = HexMultigrid(op, blk, degree=a.degree, minv=minv, blocks=blocks, coarse=a.coarse)
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t0
    info = mg.info()

    def run(M, maxiter):
        op.solve(b, M, a.tol, maxiter)                         # warm-up (graph capture, module loads)
        best = None
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            dist.barrier()
            t = time.perf_counter()
            x, si = op.solve(b, M, a.tol, maxiter)
            torch.cuda.synchronize()
            dist.barrier()
            wall = time.perf_counter() - t
            if best is None or wall < best[0]:
                best = (wall, si)
        return best

    wj, ij = run(minv, 20000)
    wm, im = run(mg, 200)
    r = b.clone()
    z = torch.empty_like(b)
    mg.apply(r, z)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.vcycles):
        mg.apply(r, z)
    e1.record()
    e1.synchronize()
    vc_ms = e0.elapsed_time(e1) / a.vcycles
    mine = {"jacobi": {"flag": ij.flag, "iters": ij.iters, "loop_ms": round(ij.loop_ms, 3), "wall_s": round(wj, 4)},
            "multigrid": {"flag": im.flag, "iters": im.iters, "loop_ms": round(im.loop_ms, 3), "wall_s": round(wm, 4),
                          "setup_s": round(setup_s, 3), "vcycle_ms": round(vc_ms, 4)}}
    box = [None] * world
    dist.all_gather_object(box, mine)
    if rank == 0:
        common = {"ranks": world, "pgrid": list(pgrid), "block": a.block, "operator": a.operator, "coarse": a.coarse, "tol": a.tol, "card": card(),
                  "shared_gpu": shared}
        print(json.dumps({**common, "arm": "jacobi", "per_rank": [m["jacobi"] for m in box]}))
        print(json.dumps({**common, "arm": "multigrid", "degree": a.degree, "levels": info["levels"], "gather_level": info["gather_level"],
                          "n_gathered": info["n_gathered"], "per_rank": [m["multigrid"] for m in box]}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
