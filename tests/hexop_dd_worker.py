"""Multi-rank worker for the index-free hex-box operator (launched by tests/test_gpu_hexop_dd.py through
torch.distributed.run; argv: out.json per field).

Every rank owns one box of partition_blocks(ng, block_grid(world)) with per^3 elements and solves the same problems on the
new operator (generate_box_operator) and on the ordered EBE operator (generate_ebe(ordered=True)), with the same halo plan:
Jacobi-PCG and, on a uniform box, MG-PCG with HexMultigrid(op, block, blocks=...).  Per rank: x, resvec and the trace
bit-identical between the two operators.  Rank 0 also checks the Jacobi solution against the oracle's multi-part
emulation of the reference.  Ranks never raise on a mismatch: they record it, and rank 0 writes every rank's findings."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist


def main():
    out_path, per, field = sys.argv[1], int(sys.argv[2]), sys.argv[3] == "1"
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    dist.init_process_group("gloo")
    from pcg_mpi_solver_b200.hexmesh import (block_field, block_grid, generate_box_operator, generate_ebe, interface_lists,
                                             load_vector, partition_blocks)
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator.from_torch_distributed(dev, nccl=False)
    pgrid = block_grid(world)
    ng = tuple(per * pgrid[a] for a in range(3))
    blocks = partition_blocks(ng, pgrid)
    for b_ in blocks:
        b_.h = 1.0 / ng[0]
    blk = blocks[rank]
    gfield = np.random.default_rng(11).uniform(0.1, 10.0, tuple(reversed(ng))) if field else None
    f = block_field(gfield, blk) if field else None
    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    b = load_vector(blk, device=dev)
    runs = {}
    for name in ("hexop", "ordered"):
        A = generate_box_operator(blk, device=dev, E_field=f) if name == "hexop" else generate_ebe(blk, device=dev, ordered=True, E_field=f)
        op = SubdomainOperator(A, comm, nbr, lists, w, n_global=n_global)
        minv = op.jacobi()
        x, info = op.solve(b, minv, 1e-11, 5000, check_every=8, record_resvec=True, trace=True)
        r = {"x": x.cpu().numpy(), "resvec": info.resvec, "trace": info.trace.tobytes(), "minv": minv.cpu().numpy(),
             "info": (info.flag, info.iters, info.relres)}
        if not field:
            mg = HexMultigrid(op, blk, blocks=blocks)
            xm, im = op.solve(b, mg, 1e-10, 200, check_every=4, record_resvec=True, trace=True)
            r.update(mx=xm.cpu().numpy(), mresvec=im.resvec, mtrace=im.trace.tobytes(), minfo=(im.flag, im.iters), lam=mg.info()["lambda"])
            del mg
        runs[name] = r
        del op, A
    h, o = runs["hexop"], runs["ordered"]
    mine = {"rank": rank, "flag": h["info"][0], "iters": h["info"][1],
            "jacobi_same": bool(np.array_equal(h["x"].view(np.uint64), o["x"].view(np.uint64)) and
                                np.array_equal(h["resvec"], o["resvec"]) and h["trace"] == o["trace"] and h["info"] == o["info"]),
            "minv_same": bool(np.array_equal(h["minv"].view(np.uint64), o["minv"].view(np.uint64)))}
    if not field:
        mine.update(mg_flag=h["minfo"][0], mg_iters=h["minfo"][1], lam_same=h["lam"] == o["lam"],
                    mg_same=bool(np.array_equal(h["mx"].view(np.uint64), o["mx"].view(np.uint64)) and
                                 np.array_equal(h["mresvec"], o["mresvec"]) and h["mtrace"] == o["mtrace"] and h["minfo"] == o["minfo"]))
    gz, gy, gx = np.meshgrid(*[np.arange(blk.e0[a], blk.e0[a] + blk.ne[a] + 1) for a in (2, 1, 0)], indexing="ij")
    keep = gx.ravel() >= 1
    gnode = ((gz * (ng[1] + 1) + gy) * (ng[0] + 1) + gx).ravel()[keep]
    gdof = (3 * gnode[:, None] + np.arange(3)[None, :]).ravel()
    gathered = [None] * world
    dist.gather_object({**mine, "gdof": gdof, "x": h["x"]}, gathered if rank == 0 else None, dst=0)
    if rank == 0:
        from oracle import ref_pcg as R
        parts = []
        for r, bl in enumerate(blocks):
            nb, ls, ww = interface_lists(blocks, r)
            if field:
                from pcg_mpi_solver_b200.hexmesh import generate_matrix
                A = generate_matrix(bl, device=dev, E_field=block_field(gfield, bl)).to_scipy()
            else:
                A = R.hex_box_csr(bl.ng, bl.e0, bl.ne, h=bl.h)
            parts.append(R.CsrPart(A, load_vector(bl, device="cpu").numpy(), nb, ls, ww, part_id=r))
        opr = R.Operator(parts)
        ref = R.ref_pcg(parts, opr.jacobi(), 1e-11, 5000, nglob=n_global)
        ntot = 3 * (ng[0] + 1) * (ng[1] + 1) * (ng[2] + 1)
        U, Uref = np.zeros(ntot), np.zeros(ntot)
        for r, g in enumerate(gathered):
            U[g["gdof"]] = g["x"]
            Uref[g["gdof"]] = ref["X"][r]
        res = {"world": world, "field": field, "transport": comm.transport, "ref_flag": ref["Flag"], "ref_iters": ref["Iter"],
               "x_rel_err": float(np.linalg.norm(U - Uref) / np.linalg.norm(Uref)),
               "ranks": [{k: v for k, v in g.items() if k not in ("gdof", "x")} for g in gathered]}
        with open(out_path, "w") as fh:
            json.dump(res, fh)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
