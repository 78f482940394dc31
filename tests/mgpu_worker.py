"""Multi-GPU parity worker (launched by tests/test_gpu_multi.py through torch.distributed.run).

Every rank owns one hex box (assembled CSR, or the matrix-free EBE operator with its separate p.q dot), solves with
the halo exchange + allreduce path and rank 0 compares
the gathered solution against the CPU oracle's multi-part emulation of the reference
(oracle/ref_pcg.py ref_pcg over CsrPart boxes with the same interface lists).  Every rank records the loop trace; rank 0
checks that the traces agree on every rank, that on the peer transport every reduced value is the rank-order sum of the
ranks' local values bit for bit, and that the host restatement of the control logic (tests/pcg_shadow.py) replays it."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist


def concrete_main(out_path, zip_path):
    """8-way METIS partition of data/concrete.zip, one part per GPU, against the reference's 8-rank run."""
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    dist.init_process_group("nccl", device_id=dev)
    from pcg_mpi_solver_b200.partition import partition_mesh
    from pcg_mpi_solver_b200.solver import Communicator
    comm = Communicator.from_torch_distributed(dev)
    gold = os.path.join(ROOT, "tests", "golden")
    ep = np.load(os.path.join(gold, f"concrete_elepart_{world}.npy")).astype(np.int64) if world == 8 else None
    subs = partition_mesh(zip_path, world, elepart=ep, assemble=False)
    sub = subs[rank]
    op = sub.to_operator(comm, device=dev)
    b = torch.from_numpy(sub.b).to(dev)
    minv = op.jacobi()
    x, info = op.solve(b, minv, 1e-7, 10000)
    gathered = [None] * world
    dist.gather_object({"gdof": sub.dof_eff_global, "x": x.cpu().numpy()}, gathered if rank == 0 else None, dst=0)
    if rank == 0:
        g = json.load(open(os.path.join(gold, "concrete_ref.json")))
        u = np.zeros(g["GlobNDof"])
        for it in gathered:
            u[it["gdof"]] = it["x"]
        s = np.load(os.path.join(gold, "concrete_ref_samples.npz"))
        key = f"U{world}" if f"U{world}" in s else "U1"
        res = {"world": world, "flag": info.flag, "iters": info.iters, "relres": info.relres, "norm_u": float(np.linalg.norm(u)),
               "ref": g["runs"].get(str(world), g["runs"]["1"]), "sample_err": float(np.abs(u[s["idx"]] - s[key]).max() / np.abs(s[key]).max()),
               "loop_ms": info.loop_ms, "halo_bytes": op.halo_bytes()}
        json.dump(res, open(out_path, "w"))
        print(json.dumps({k: v for k, v in res.items() if k != "ref"}))
    dist.barrier()
    dist.destroy_process_group()


# slots of the trace records that hold a reduced value with a local counterpart, per record kind
_REDUCED_SLOTS = {0: (4, 5), 1: (0, 1, 2, 3, 4, 5), 2: (3,), 3: (4, 5), 4: (3,)}


def trace_checks(gathered, transport, tol, maxiter, n_global):
    """Rank-0 checks of the traces of all ranks."""
    from tests import pcg_shadow as S
    traces = [g["trace"] for g in gathered]
    out = {"trace_records": len(traces[0]), "trace_complete": all(g["trace_total"] == len(g["trace"]) for g in gathered)}
    ranks_ok = [all(int(r) == k for r in t["rank"]) for k, t in enumerate(traces)]

    def shared_part(t):
        t = t.copy()
        t["rank"] = 0
        t["local"] = 0.0
        return t.tobytes()

    out["trace_identical"] = all(ranks_ok) and all(shared_part(t) == shared_part(traces[0]) for t in traces)
    checked = mismatches = 0
    if transport == "peer" and out["trace_identical"]:
        for j, rec in enumerate(traces[0]):
            for slot in _REDUCED_SLOTS[int(rec["kind"])]:
                s = 0.0
                for t in traces:          # the peer all-reduce adds the ranks' values in rank order, starting from 0
                    s = s + float(t[j]["local"][slot])
                checked += 1
                mismatches += 0 if S.same_bits(s, float(rec["inp"][slot])) else 1
    out["trace_sum_checked"], out["trace_sum_mismatches"] = checked, mismatches
    try:
        S.replay(traces[0], tol, maxiter, n_global)
        out["trace_replayed"] = True
    except AssertionError as e:
        out["trace_replayed"] = str(e)[:300]
    return out


def main():
    out_path = sys.argv[1]
    if len(sys.argv) > 2 and sys.argv[2] == "concrete":
        return concrete_main(out_path, sys.argv[3])
    block = int(sys.argv[2]) if len(sys.argv) > 2 else 6
    use_graph = bool(int(sys.argv[3])) if len(sys.argv) > 3 else True
    operator = sys.argv[4] if len(sys.argv) > 4 else "csr"      # csr | ebe (matrix-free, fp64-atomic scatter) | ebe_ordered
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    # PCGB_SHARED_GPU=1: all ranks drive cuda:0 (time-sliced) with a peer-only communicator - exercises the peer-memory
    # halo / all-reduce kernels between OS processes on a ONE-GPU box (NCCL refuses two ranks on one device)
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    from pcg_mpi_solver_b200.hexmesh import (block_grid, generate_ebe, generate_matrix, interface_lists, load_vector,
                                             partition_blocks)
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    if os.environ.get("PCGB_EXPECT_TRANSPORT"):
        assert comm.transport == os.environ["PCGB_EXPECT_TRANSPORT"], (comm.transport, comm.peer_error)
    pgrid = block_grid(world)
    ng = tuple(block * pgrid[a] + (1 if a == 1 else 0) for a in range(3))  # uneven cut along y
    blocks = partition_blocks(ng, pgrid)
    for b_ in blocks:
        b_.h = 1.0 / ng[0]
    blk = blocks[rank]
    A = generate_matrix(blk, device=dev) if operator == "csr" else generate_ebe(blk, device=dev, ordered=operator == "ebe_ordered")
    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    op = SubdomainOperator(A, comm, nbr, lists, w, n_global=n_global)
    b = load_vector(blk, device=dev)
    minv = op.jacobi()
    tol = float(sys.argv[5]) if len(sys.argv) > 5 else 1e-12
    x, info = op.solve(b, minv, tol, 5000, use_graph=use_graph, check_every=8, trace=True)
    # operator probe: y = K v for a globally consistent v (function of the global dof id)
    gz, gy, gx = np.meshgrid(*[np.arange(blk.e0[a], blk.e0[a] + blk.ne[a] + 1) for a in (2, 1, 0)], indexing="ij")
    keep = gx.ravel() >= 1
    gnode = ((gz * (ng[1] + 1) + gy) * (ng[0] + 1) + gx).ravel()[keep]
    gdof = (3 * gnode[:, None] + np.arange(3)[None, :]).ravel()
    v = np.sin(0.37 * gdof) + 0.01 * (gdof % 7)
    y = op.apply(torch.from_numpy(v).to(dev)).cpu().numpy()
    wsum = torch.tensor([float(np.sum(w))], dtype=torch.float64, device=dev)
    comm.allreduce_sum(wsum)
    # a second operator application AFTER the solve: the exchange epochs keep counting across graph replays and direct calls
    y2 = op.apply(torch.from_numpy(v).to(dev)).cpu().numpy()
    if operator != "ebe":
        assert np.array_equal(y, y2), "operator application is not reproducible"
    else:                                                         # atomics: reproducible to rounding only
        assert np.abs(y - y2).max() <= 1e-14 * np.abs(y).max(), "operator application is not reproducible"
    gathered = [None] * world
    dist.gather_object({"gdof": gdof, "x": x.cpu().numpy(), "y": y, "w": w, "info": (info.flag, info.iters, info.relres),
                        "trace": info.trace, "trace_total": info.trace_total,
                        "x_sha": hashlib.sha256(x.cpu().numpy().tobytes()).hexdigest(),
                        "trace_sha": hashlib.sha256(info.trace.tobytes()).hexdigest(),
                        "halo_m": op.halo_bytes() // 8, "halo_ndof": int(len(np.unique(np.concatenate(lists)))) if len(lists) else 0},
                       gathered if rank == 0 else None, dst=0)
    if rank == 0:
        from oracle import ref_pcg as R
        parts = []
        for r, bl in enumerate(blocks):
            nb, ls, ww = interface_lists(blocks, r)
            Ar = R.hex_box_csr(bl.ng, bl.e0, bl.ne, h=bl.h)
            br = load_vector(bl, device="cpu").numpy()
            parts.append(R.CsrPart(Ar, br, nb, ls, ww, part_id=r))
        opr = R.Operator(parts)
        ref = R.ref_pcg(parts, opr.jacobi(), tol, 5000, nglob=n_global)
        ntot = 3 * (ng[0] + 1) * (ng[1] + 1) * (ng[2] + 1)
        U, Uref, Y, Yref = (np.zeros(ntot) for _ in range(4))
        yrefs = opr.apply([np.sin(0.37 * g["gdof"]) + 0.01 * (g["gdof"] % 7) for g in gathered])
        consistent = 0.0
        for r, g in enumerate(gathered):
            # copies of shared dofs must agree between ranks (consistent vectors)
            seen = U[g["gdof"]] != 0
            if seen.any():
                consistent = max(consistent, float(np.abs(U[g["gdof"]][seen] - g["x"][seen]).max()))
            U[g["gdof"]] = g["x"]
            Uref[g["gdof"]] = ref["X"][r]
            Y[g["gdof"]] = g["y"]
            Yref[g["gdof"]] = yrefs[r]
        res = {**trace_checks(gathered, comm.transport, tol, 5000, n_global),
               "world": world, "tol": tol, "flag": info.flag, "iters": info.iters, "relres": info.relres, "ref_flag": ref["Flag"],
               "ref_iters": ref["Iter"], "ref_relres": ref["RelRes"],
               "x_rel_err": float(np.linalg.norm(U - Uref) / np.linalg.norm(Uref)),
               "y_rel_err": float(np.linalg.norm(Y - Yref) / np.linalg.norm(Yref)),
               "copy_mismatch": consistent / float(np.abs(U).max()), "weight_sum": float(wsum.item()), "n_global": n_global,
               "halo_bytes": op.halo_bytes(), "all_infos": [g["info"] for g in gathered], "transport": comm.transport,
               "x_sha": [g["x_sha"] for g in gathered], "trace_sha": [g["trace_sha"] for g in gathered],
               "halo_m": [g["halo_m"] for g in gathered], "halo_ndof": [g["halo_ndof"] for g in gathered],
               "plan": A.plan_info() if operator == "csr" else "ebe", "launches": info.launches, "loop_ms": info.loop_ms}
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
