"""Compare the three operators of the 128^3 hex box on one GPU: assembled CSR, matrix-free EBE (fp64-atomic scatter) and
the ordered matrix-free EBE operator (fixed summation order, bit-reproducible).

Per operator: PCG iterations per second over a fixed number of device-timed iterations (info.loop_ms, after a warm-up
solve; the three operators alternate, `--repeats` rounds), ms per operator application from a time_kernels pass, the
peak device memory while the operator is built and solved, and the algorithmic bytes per application.  Parity: the
ordered operator's residual history against tests/golden/hex128_N1_resvec.json and the x of two of its runs bit for
bit.  The GPU name and power limit come from a read-only nvidia-smi query.  With oracle/_ref/concrete.zip staged, one
concrete solve to 1e-8 with the ordered operator.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (s.strip() for s in out[0].split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:     # the measurement still stands; the card is then named by torch alone
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": None, "nvidia_smi_error": str(e)[:200]}


def build(kind, blk, dev):
    from pcg_mpi_solver_b200.hexmesh import generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    free0, _ = torch.cuda.mem_get_info(dev)
    if kind == "csr":
        M = generate_matrix(blk, device=dev)
    else:
        M = generate_ebe(blk, device=dev, ordered=(kind == "ebe_ordered"))
    op = SubdomainOperator(M)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info(dev)
    # torch-owned tensors (CSR arrays, element indices) show in the allocator; library allocations (plans, slot buffer,
    # slot lists, solver vectors) only in the device's free memory
    return M, op, {"torch_peak_bytes": torch.cuda.max_memory_allocated(dev) - base, "device_bytes_used": free0 - free1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ebe_ordered_bench: needs a CUDA device")
    from pcg_mpi_solver_b200.hexmesh import HexBlock, load_vector
    dev = torch.device("cuda:0")
    B = a.block
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    b = load_vector(blk, device=dev)
    kinds = ("csr", "ebe", "ebe_ordered")
    ops, out = {}, {"block": B, "n": blk.n, "steps": a.steps, "warmup": a.warmup, **gpu_info()}
    for k in kinds:
        M, op, mem = build(k, blk, dev)
        ops[k] = (M, op, op.jacobi())
        out[k] = {**mem, "bytes_per_apply": int(M.spmv_bytes()), "it_per_s": []}
    for _ in range(a.repeats):                                         # alternate the operators
        for k in kinds:
            M, op, minv = ops[k]
            op.solve(b, minv, 0.0, a.warmup, fixed_iters=True, check_every=a.warmup)
            _, info = op.solve(b, minv, 0.0, a.steps, fixed_iters=True, check_every=50)
            out[k]["it_per_s"].append(a.steps / (info.loop_ms * 1e-3))
    for k in kinds:
        M, op, minv = ops[k]
        _, info = op.solve(b, minv, 0.0, 50, fixed_iters=True, time_kernels=True)
        out[k]["ms_per_apply"] = info.phase_ms["spmv"]
        out[k]["ms_per_iteration"] = info.phase_ms["iteration"]
        out[k]["it_per_s_median"] = float(np.median(out[k]["it_per_s"]))
        out[k]["GBps_algorithmic"] = out[k]["bytes_per_apply"] / (info.phase_ms["spmv"] * 1e-3) / 1e9
    # parity of the ordered operator
    M, op, minv = ops["ebe_ordered"]
    gold_path = os.path.join(ROOT, "tests", "golden", f"hex{B}_N1_resvec.json")
    x1, i1 = op.solve(b, minv, 0.0, 40, fixed_iters=True, record_resvec=True, check_every=20)
    x2, i2 = op.solve(b, minv, 0.0, 40, fixed_iters=True, record_resvec=True, check_every=20)
    par = {"x_bit_identical_two_runs": bool(torch.equal(x1, x2)), "resvec_bit_identical": bool(np.array_equal(i1.resvec, i2.resvec))}
    if os.path.exists(gold_path):
        ref = np.array(json.load(open(gold_path))["resvec"])
        m = min(len(ref), len(i1.resvec))
        par["resvec_max_rel_err_vs_golden"] = float(np.max(np.abs(i1.resvec[:m] - ref[:m]) / ref[:m]))
        par["resvec_compared"] = m
    xs = torch.randn(blk.n, dtype=torch.float64, device=dev)
    yc = ops["csr"][0].spmv(xs)
    for k in ("ebe", "ebe_ordered"):
        par[f"{k}_vs_csr_max_rel"] = float((ops[k][0].apply_local(xs) - yc).abs().max() / yc.abs().max())
    out["ebe_ordered_parity"] = par
    del ops, M, op, minv
    zp = os.path.join(ROOT, "oracle", "_ref", "concrete.zip")
    if os.path.exists(zp):
        from pcg_mpi_solver_b200.partition import partition_mesh
        sub = partition_mesh(zp, 1, assemble=False)[0]
        cop = sub.to_operator(device=dev, kind="ebe_ordered")
        _, info = cop.solve(torch.from_numpy(sub.b).to(dev), cop.jacobi(), 1e-8, 20000)
        out["concrete_ebe_ordered"] = {"flag": info.flag, "iters": info.iters, "relres": info.relres, "loop_ms": info.loop_ms}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
