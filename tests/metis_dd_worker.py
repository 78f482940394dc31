"""Multi-rank worker on element-partitioned models (launched by tests/test_gpu_metis_dd.py through torch.distributed.run).

argv: output json, model (`concrete` or `hex:<case>` of tests/metis_dd_cases.py), partition (`golden` = the reference's
8-way split of concrete, `metis` = run_metis, or the hex case's own), operator (`csr` = device assembly, `ebe`,
`ebe_ordered`), graph (0/1), tol, maxiter, and the maxiter of the reproducibility solves (0 = maxiter).

Every rank builds `partition_mesh(model, world, elepart, assemble=False)[rank]` and `sub.to_operator(comm, device, kind)`,
then checks, recording mismatches instead of raising so that all ranks stay in step (rank 0 writes everything):
- the exchange bit for bit: op.exchange_add(y_r) of the local product y_r of a consistent probe v against the host
  exchange (tests/metis_dd_cases.exchange) of every rank's y_r;
- op.apply(v) against that exchanged local product, bit for bit (within 1e-13 (|A||v|) for the atomic `ebe`);
- op.jacobi() against 1 / exchange(diag_r), bit for bit;
- the product against a reference: on hex, oracle.ref_pcg.Operator over host-assembled CsrParts with the same lists,
  entrywise within 1e-13 (|A||v|); on concrete, the reference's own calcMPFint and updatePreconditioner probe;
- Jacobi-PCG with the trace (mgpu_worker.trace_checks), copies of shared dofs, the weight sum, and against ref_pcg (hex)
  or the reference's own run (concrete);
- csr and ebe_ordered: graph on/off x check_every 1/7 give bit-identical x and trace."""
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

from tests import metis_dd_cases as C


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    out_path, model_arg, part_arg, kind = sys.argv[1:5]
    graph, tol, maxiter = bool(int(sys.argv[5])), float(sys.argv[6]), int(sys.argv[7])
    repro_maxiter = int(sys.argv[8]) if len(sys.argv) > 8 and int(sys.argv[8]) > 0 else maxiter
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"     # all ranks on cuda:0, peer-only communicator
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    t0 = time.time()
    from pcg_mpi_solver_b200.model import load_mdf
    from pcg_mpi_solver_b200.partition import build_subdomains
    from pcg_mpi_solver_b200.solver import Communicator
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    if os.environ.get("PCGB_EXPECT_TRANSPORT"):
        assert comm.transport == os.environ["PCGB_EXPECT_TRANSPORT"], (comm.transport, comm.peer_error)
    concrete = model_arg == "concrete"
    if concrete:
        model = load_mdf(C.CONCRETE_ZIP)
        if part_arg == "golden":
            ep = np.load(os.path.join(C.GOLD, f"concrete_elepart_{world}.npy")).astype(np.int64)
        else:                                   # METIS on rank 0, the same split everywhere
            from pcg_mpi_solver_b200.metis import run_metis
            box = [run_metis(model.node_flat, model.node_offset, world) if rank == 0 else None]
            dist.broadcast_object_list(box, src=0)
            ep = box[0]
    else:
        case = model_arg.split(":", 1)[1]
        assert C.CASES[case][1] == world, (case, world)
        model = C.hex_model(case)
        ep = C.elepart(case, model)
    subs = build_subdomains(model, ep, world, assemble=False)
    sub = subs[rank]
    op = sub.to_operator(comm, dev, kind)
    tables = [(s.id, s.nbr, s.ovrlp) for s in subs]
    fails = []

    def t(v):
        return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)

    def allgather(obj):
        box = [None] * world
        dist.all_gather_object(box, obj)
        return box

    def check_bits(what, got, want):
        if not C.same_bits(got, want):
            bad = int(np.sum(np.asarray(got) != np.asarray(want))) if np.shape(got) == np.shape(want) else -1
            fails.append(f"rank {rank} {what}: {bad} of {np.size(want)} entries differ")

    gdof = sub.dof_eff_global
    v = C.probe(gdof, concrete)
    # ---- exchange, apply and Jacobi, bit for bit against the host exchange of every rank's local values
    y_loc = (op.A.spmv(t(v)) if kind == "csr" else op.A.apply_local(t(v))).cpu().numpy()
    diag = op.A.diagonal().cpu().numpy()
    bound_loc = C.abs_product(sub, v)
    every = allgather({"y": y_loc, "d": diag, "bound": bound_loc})
    y_want = C.exchange(tables, [e["y"] for e in every])[rank]
    bound = C.exchange(tables, [e["bound"] for e in every])[rank]
    check_bits("exchange_add", op.exchange_add(t(y_loc)).cpu().numpy(), y_want)
    y_app = op.apply(t(v)).cpu().numpy()
    if kind == "ebe":                           # fp64 atomics: the local product is reproducible to rounding only
        if not np.all(np.abs(y_app - y_want) <= 1e-13 * bound):
            fails.append(f"rank {rank} apply: off the exchanged local product by more than 1e-13 (|A||v|)")
    else:
        check_bits("apply", y_app, y_want)
    minv = op.jacobi()
    check_bits("jacobi", minv.cpu().numpy(), 1.0 / C.exchange(tables, [e["d"] for e in every])[rank])
    # ---- Jacobi-PCG with the trace; with csr and ebe_ordered, graph on/off x check_every 1/7 give the same bits
    b = t(sub.b)
    x, info = op.solve(b, minv, tol, maxiter, use_graph=graph, check_every=8, trace=True)
    xs = x.cpu().numpy()
    wsum = torch.tensor([float(np.sum(sub.weights))], dtype=torch.float64, device=dev)
    comm.allreduce_sum(wsum)
    repro = []
    if kind != "ebe":
        for g_ in (0, 1):
            for ce in (1, 7):
                xr, ir = op.solve(b, minv, tol, repro_maxiter, use_graph=bool(g_), check_every=ce, trace=True)
                repro.append({"graph": g_, "check_every": ce, "x_sha": _sha(xr.cpu().numpy()), "trace_sha": _sha(ir.trace),
                              "info": (ir.flag, ir.iters, ir.relres)})
    y2 = op.apply(t(v)).cpu().numpy()           # after the solves: the exchange epochs keep counting across graph replays
    if kind != "ebe":
        check_bits("apply after the solves", y2, y_app)
    torch.cuda.synchronize()
    from pcg_mpi_solver_b200 import _lib
    status = _lib.load().pcgb_comm_status(comm.handle, _lib.stream_ptr())
    if status != 0:
        fails.append(f"rank {rank}: communicator status {status}")
    gathered = [None] * world
    dist.gather_object({"gdof": gdof, "x": xs, "y": y_app, "minv": minv.cpu().numpy(), "bound": bound, "fails": fails,
                        "info": (info.flag, info.iters, info.relres), "trace": info.trace, "trace_total": info.trace_total,
                        "x_sha": _sha(xs), "trace_sha": _sha(info.trace), "repro": repro, "halo_m": op.halo_bytes() // 8,
                        "plan": op.A.plan_info() if kind == "csr" else None, "seconds": time.time() - t0,
                        "loop_ms": info.loop_ms}, gathered if rank == 0 else None, dst=0)
    if rank == 0:
        from tests.mgpu_worker import trace_checks
        n_global = sub.n_global_eff
        res = {**trace_checks(gathered, comm.transport, tol, maxiter, n_global), "world": world, "model": model_arg,
               "partition": part_arg, "operator": kind, "graph": graph, "tol": tol, "maxiter": maxiter, "transport": comm.transport,
               "flag": info.flag, "iters": info.iters, "relres": info.relres, "all_infos": [g["info"] for g in gathered],
               "weight_sum": float(wsum.item()), "n_global": n_global, "fails": [f for g in gathered for f in g["fails"]],
               "x_sha": [g["x_sha"] for g in gathered], "trace_sha": [g["trace_sha"] for g in gathered],
               "repro": [g["repro"] for g in gathered], "halo_m": [g["halo_m"] for g in gathered],
               "plan": [g["plan"] for g in gathered], "seconds": max(g["seconds"] for g in gathered),
               "loop_ms": max(g["loop_ms"] for g in gathered)}
        # copies of shared dofs must agree between ranks
        U = np.zeros(model.n_dof)
        seen = np.zeros(model.n_dof, dtype=bool)
        copy = 0.0
        for g in gathered:
            s = seen[g["gdof"]]
            if s.any():
                copy = max(copy, float(np.abs(U[g["gdof"]][s] - g["x"][s]).max()))
            U[g["gdof"]] = g["x"]
            seen[g["gdof"]] = True
        res["copy_mismatch"] = copy / max(float(np.abs(U).max()), 1e-300)
        if concrete:
            arr = np.load(os.path.join(C.GOLD, "concrete_probe.npz"))
            gold = json.load(open(os.path.join(C.GOLD, "concrete_ref.json")))
            Y = C.gather(model.n_dof, [g["gdof"] for g in gathered], [g["y"] for g in gathered])
            free = np.isin(arr["idx"], model.dof_eff)
            res["probe_dofs"] = int(free.sum())
            res["probe_y_ok"] = bool(np.allclose(Y[arr["idx"][free]], arr["y"][free], rtol=1e-12, atol=1e-9 * np.abs(arr["y"]).max()))
            Minv = C.gather(model.n_dof, [g["gdof"] for g in gathered], [g["minv"] for g in gathered])
            res["probe_minv_ok"] = bool(np.allclose(Minv[model.dof_eff[arr["minv_idx"]]], arr["minv"], rtol=1e-13, atol=0.0))
            samples = np.load(os.path.join(C.GOLD, "concrete_ref_samples.npz"))
            key = f"U{world}" if part_arg == "golden" else "U1"
            res["ref"] = {k: v_ for k, v_ in gold["runs"][str(world) if part_arg == "golden" else "1"].items() if k != "parts"}
            res["norm_u"] = float(np.linalg.norm(U))
            res["sample_err"] = float(np.abs(U[samples["idx"]] - samples[key]).max() / np.abs(samples[key]).max())
        else:
            from oracle import ref_pcg as R
            hsubs = build_subdomains(model, ep, world, assemble=True)
            parts = [R.CsrPart(s.A, s.b, s.nbr, s.ovrlp, s.weights, part_id=s.id) for s in hsubs]
            opr = R.Operator(parts)
            yref = opr.apply([C.probe(s.dof_eff_global) for s in hsubs])
            res["y_entry_ok"] = all(bool(np.all(np.abs(g["y"] - yr) <= 1e-13 * g["bound"])) for g, yr in zip(gathered, yref))
            res["y_rel_err"] = max(float(np.abs(g["y"] - yr).max() / np.abs(yr).max()) for g, yr in zip(gathered, yref))
            # and against the product of the whole model on one part, which does not depend on the interface lists
            one = build_subdomains(model, np.zeros(model.n_elem, dtype=np.int64), 1, assemble=True)[0]
            vg = C.probe(one.dof_eff_global)
            Yg, Bg = np.zeros(model.n_dof), np.zeros(model.n_dof)
            Yg[one.dof_eff_global], Bg[one.dof_eff_global] = one.A @ vg, abs(one.A) @ np.abs(vg)
            res["y_global_ok"] = all(bool(np.all(np.abs(g["y"] - Yg[g["gdof"]]) <= 1e-13 * Bg[g["gdof"]])) for g in gathered)
            ref = R.ref_pcg(parts, opr.jacobi(), tol, maxiter, nglob=n_global)
            Uref = C.gather(model.n_dof, [g["gdof"] for g in gathered], ref["X"])
            res.update(ref_flag=ref["Flag"], ref_iters=ref["Iter"], ref_relres=ref["RelRes"],
                       x_rel_err=float(np.linalg.norm(U - Uref) / np.linalg.norm(Uref)))
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps({k: v_ for k, v_ in res.items() if k not in ("repro", "x_sha", "trace_sha", "plan")}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
