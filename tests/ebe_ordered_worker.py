"""Multi-rank worker for the ordered matrix-free operator (launched by tests/test_gpu_ebe_ordered.py through
torch.distributed.run).

Every rank owns one hex box as an EbeMatrixOrdered and solves twice with the halo exchange + all-reduce path; rank 0
checks both solutions against the CPU oracle's multi-part emulation of the reference, that the two runs gave the same
bits on every rank, that operator applications repeat bit for bit, and the loop traces (tests/mgpu_worker.trace_checks)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist


def main():
    out_path = sys.argv[1]
    block = int(sys.argv[2])
    use_graph = bool(int(sys.argv[3]))
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"     # all ranks on cuda:0 over the peer transport
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    from pcg_mpi_solver_b200.hexmesh import block_grid, generate_ebe, interface_lists, load_vector, partition_blocks
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    from tests.mgpu_worker import trace_checks
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    if os.environ.get("PCGB_EXPECT_TRANSPORT"):
        assert comm.transport == os.environ["PCGB_EXPECT_TRANSPORT"], (comm.transport, comm.peer_error)
    pgrid = block_grid(world)
    ng = tuple(block * pgrid[a] + (1 if a == 1 else 0) for a in range(3))  # uneven cut along y
    blocks = partition_blocks(ng, pgrid)
    for b_ in blocks:
        b_.h = 1.0 / ng[0]
    blk = blocks[rank]
    E = generate_ebe(blk, device=dev, ordered=True)
    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    op = SubdomainOperator(E, comm, nbr, lists, w, n_global=n_global)
    b = load_vector(blk, device=dev)
    minv = op.jacobi()
    tol = 1e-12
    x, info = op.solve(b, minv, tol, 5000, use_graph=use_graph, check_every=8, trace=True)
    x2, info2 = op.solve(b, minv, tol, 5000, use_graph=use_graph, check_every=8, record_resvec=True)
    gz, gy, gx = np.meshgrid(*[np.arange(blk.e0[a], blk.e0[a] + blk.ne[a] + 1) for a in (2, 1, 0)], indexing="ij")
    keep = gx.ravel() >= 1
    gnode = ((gz * (ng[1] + 1) + gy) * (ng[0] + 1) + gx).ravel()[keep]
    gdof = (3 * gnode[:, None] + np.arange(3)[None, :]).ravel()
    v = np.sin(0.37 * gdof) + 0.01 * (gdof % 7)
    y = op.apply(torch.from_numpy(v).to(dev)).cpu().numpy()
    y2 = op.apply(torch.from_numpy(v).to(dev)).cpu().numpy()
    gathered = [None] * world
    dist.gather_object({"gdof": gdof, "x": x.cpu().numpy(), "same_x": bool(torch.equal(x, x2)), "same_y": bool(np.array_equal(y, y2)),
                        "y": y, "info": (info.flag, info.iters, info.relres), "info2": (info2.flag, info2.iters, info2.relres),
                        "trace": info.trace, "trace_total": info.trace_total},
                       gathered if rank == 0 else None, dst=0)
    if rank == 0:
        from oracle import ref_pcg as R
        parts = []
        for r, bl in enumerate(blocks):
            nb, ls, ww = interface_lists(blocks, r)
            parts.append(R.CsrPart(R.hex_box_csr(bl.ng, bl.e0, bl.ne, h=bl.h), load_vector(bl, device="cpu").numpy(), nb, ls, ww, part_id=r))
        opr = R.Operator(parts)
        ref = R.ref_pcg(parts, opr.jacobi(), tol, 5000, nglob=n_global)
        ntot = 3 * (ng[0] + 1) * (ng[1] + 1) * (ng[2] + 1)
        U, Uref, Y, Yref = (np.zeros(ntot) for _ in range(4))
        yrefs = opr.apply([np.sin(0.37 * g["gdof"]) + 0.01 * (g["gdof"] % 7) for g in gathered])
        for r, g in enumerate(gathered):
            U[g["gdof"]] = g["x"]
            Uref[g["gdof"]] = ref["X"][r]
            Y[g["gdof"]] = g["y"]
            Yref[g["gdof"]] = yrefs[r]
        res = {**trace_checks(gathered, comm.transport, tol, 5000, n_global),
               "world": world, "flag": info.flag, "iters": info.iters, "relres": info.relres, "ref_flag": ref["Flag"],
               "ref_iters": ref["Iter"], "x_rel_err": float(np.linalg.norm(U - Uref) / np.linalg.norm(Uref)),
               "y_rel_err": float(np.linalg.norm(Y - Yref) / np.linalg.norm(Yref)),
               "same_x_all_ranks": all(g["same_x"] for g in gathered), "same_y_all_ranks": all(g["same_y"] for g in gathered),
               "all_infos": [g["info"] for g in gathered] + [g["info2"] for g in gathered], "transport": comm.transport,
               "loop_ms": info.loop_ms}
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
