"""The index-free hex-box operator (HexBoxOperator, csrc/hexop.cuh) against the assembled CSR matrix and the ordered EBE
operator on one GPU.

    python tools/hexop_bench.py [--block 128] [--steps 200] [--warmup 20] [--repeats 3] [--large 640,512] [--mg-large]

- 128^3 (--block), uniform and an inclusion_field voxel box at contrast 100: per operator PCG iterations/s over --steps
  device-timed iterations (the three operators alternate, --repeats rounds), ms per application from a time_kernels pass,
  algorithmic bytes and FLOPs per application with the share of the HBM and FP64 floors (data-sheet 3.35 TB/s and 34
  TFLOP/s non-tensor FP64 of an H100 SXM at 700 W) and which bounds, and the device memory the operator and its solver
  take.
- Multigrid: MG-PCG to 1e-8 (HexMultigrid, degree 2) with the new fine operator against the ordered one: iterations,
  V-cycle ms, wall time.
- Parity: the new operator's residual history against tests/golden/hex<B>_N1_resvec.json (exit status 1 above 1e-9 over
  the first 11 entries), and x, resvec and the loop trace bit-identical to the ordered operator's 40 iterations.
- Large boxes (--large): 20 fixed Jacobi-PCG iterations on the new operator, ms per iteration and the drop in free device
  memory; --mg-large also builds HexMultigrid(coarse="index_free") on each large box and times MG-PCG to --tol on it:
  iterations, flag, wall time (best of two after a warm-up solve), set-up time, V-cycle ms, info()["bytes"] against
  multigrid.index_free_bytes, the drop in free device memory across the set-up and the true relative residual.
Prints one JSON line with the card's name, power limit and SM clock limit, read in the same call."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

HBM_BPS, FP64_FLOPS = 3.35e12, 34e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (s.strip() for s in out[0].split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:     # the measurement still stands; the card is then named by torch alone
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": None, "nvidia_smi_error": str(e)[:200]}


def _free(dev):
    gc.collect()
    torch.cuda.synchronize(dev)
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(dev)[0]


def build(kind, blk, dev, field):
    from pcg_mpi_solver_b200.hexmesh import generate_box_operator, generate_ebe, generate_matrix
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    free0 = _free(dev)
    if kind == "csr":
        M = generate_matrix(blk, device=dev, E_field=field)
    elif kind == "ebe_ordered":
        M = generate_ebe(blk, device=dev, ordered=True, E_field=field)
    else:
        M = generate_box_operator(blk, device=dev, E_field=field)
    op = SubdomainOperator(M)
    minv = op.jacobi()
    free1 = _free(dev)
    return M, op, minv, free0 - free1


def compare(blk, dev, field, a):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    b = load_vector(blk, device=dev)
    kinds = ("csr", "ebe_ordered", "hexop")
    ops, out = {}, {}
    ne = int(np.prod(blk.ne))
    for k in kinds:
        M, op, minv, used = build(k, blk, dev, field)
        ops[k] = (M, op, minv)
        out[k] = {"device_bytes_operator_and_solver": int(used), "bytes_per_apply": int(M.spmv_bytes()), "it_per_s": []}
    for _ in range(a.repeats):
        for k in kinds:
            M, op, minv = ops[k]
            op.solve(b, minv, 0.0, a.warmup, fixed_iters=True, check_every=a.warmup)
            _, info = op.solve(b, minv, 0.0, a.steps, fixed_iters=True, check_every=50)
            out[k]["it_per_s"].append(round(a.steps / (info.loop_ms * 1e-3), 1))
    flops = 2 * 576 * ne                        # the element products' FMAs (the same for both matrix-free operators)
    for k in kinds:
        M, op, minv = ops[k]
        _, info = op.solve(b, minv, 0.0, 50, fixed_iters=True, time_kernels=True)
        ms = info.phase_ms["spmv"]
        r = out[k]
        r["ms_per_apply"] = round(ms, 4)
        r["ms_per_iteration"] = round(info.phase_ms["iteration"], 4)
        r["it_per_s_median"] = float(np.median(r["it_per_s"]))
        r["launches_per_solve_50"] = int(info.launches)
        if k != "csr":
            t_hbm, t_fp = r["bytes_per_apply"] / HBM_BPS * 1e3, flops / FP64_FLOPS * 1e3
            r.update(flops_per_apply=flops, hbm_floor_ms=round(t_hbm, 4), fp64_floor_ms=round(t_fp, 4),
                     bound="fp64" if t_fp >= t_hbm else "hbm", share_of_floor=round(max(t_hbm, t_fp) / ms, 3))
    del ops
    return out


def parity(blk, dev, B):
    from pcg_mpi_solver_b200.hexmesh import generate_box_operator, generate_ebe, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    b = load_vector(blk, device=dev)
    runs = []
    for kind in ("hexop", "ebe_ordered"):
        _free(dev)
        A = generate_box_operator(blk, device=dev) if kind == "hexop" else generate_ebe(blk, device=dev, ordered=True)
        op = SubdomainOperator(A)
        runs.append(op.solve(b, op.jacobi(), 0.0, 40, fixed_iters=True, record_resvec=True, check_every=20, trace=True))
        del op, A
    (xh, ih), (xo, io) = runs
    par = {"x_bit_identical_to_ordered": bool(torch.equal(xh, xo)),
           "resvec_bit_identical_to_ordered": bool(np.array_equal(ih.resvec, io.resvec)),
           "trace_bit_identical_to_ordered": ih.trace.tobytes() == io.trace.tobytes()}
    gold_path = os.path.join(ROOT, "tests", "golden", f"hex{B}_N1_resvec.json")
    ok = par["x_bit_identical_to_ordered"] and par["resvec_bit_identical_to_ordered"] and par["trace_bit_identical_to_ordered"]
    if os.path.exists(gold_path):
        ref = np.array(json.load(open(gold_path))["resvec"])
        m = min(len(ref), len(ih.resvec))
        rel = np.abs(ih.resvec[:m] - ref[:m]) / ref[:m]
        par.update(resvec_max_rel_err_vs_golden_first11=float(rel[:11].max()), resvec_max_rel_err_vs_golden=float(rel.max()),
                   resvec_compared=m)
        ok = ok and rel[:11].max() <= 1e-9
    par["ok"] = bool(ok)
    return par


def multigrid(blk, dev, tol):
    from pcg_mpi_solver_b200.hexmesh import generate_box_operator, generate_ebe, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    b = load_vector(blk, device=dev)
    out = {}
    for kind in ("hexop", "ebe_ordered"):
        _free(dev)
        A = generate_box_operator(blk, device=dev) if kind == "hexop" else generate_ebe(blk, device=dev, ordered=True)
        op = SubdomainOperator(A)
        mg = HexMultigrid(op, blk)
        op.solve(b, mg, tol, 200)
        best = None
        for _ in range(3):
            torch.cuda.synchronize()
            t = time.perf_counter()
            x, si = op.solve(b, mg, tol, 200)
            torch.cuda.synchronize()
            w = time.perf_counter() - t
            best = w if best is None else min(best, w)
        z = torch.empty_like(b)
        mg.apply(b, z)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            mg.apply(b, z)
        e1.record()
        e1.synchronize()
        out[kind] = {"flag": si.flag, "iters": si.iters, "wall_s": round(best, 4), "loop_ms": round(si.loop_ms, 3),
                     "vcycle_ms": round(e0.elapsed_time(e1) / 20, 4), "x": x}
        del mg, op, A
    out["x_bit_identical"] = bool(torch.equal(out["hexop"].pop("x"), out["ebe_ordered"].pop("x")))
    return out


def large_mg(blk, op, b, minv, dev, tol):
    """MG-PCG to tol with the index-free hierarchy on a large box (HexMultigrid(coarse="index_free"))."""
    from pcg_mpi_solver_b200.multigrid import HexMultigrid, index_free_bytes
    free0 = _free(dev)
    try:
        t = time.perf_counter()
        mg = HexMultigrid(op, blk, minv=minv, coarse="index_free")
        torch.cuda.synchronize()
        setup = time.perf_counter() - t
    except Exception as e:
        return {"fits": False, "error": str(e)[:200], "index_free_bytes": index_free_bytes(blk.ne), "free_before_bytes": int(free0)}
    info = mg.info()
    r = {"fits": True, "setup_s": round(setup, 3), "bytes": info["bytes"], "index_free_bytes": index_free_bytes(blk.ne),
         "free_drop_bytes": int(free0 - torch.cuda.mem_get_info(dev)[0]), "levels": info["levels"]}
    op.solve(b, mg, tol, 100)                                  # warm-up (graph capture, module loads)
    best = None
    for _ in range(2):
        torch.cuda.synchronize()
        t = time.perf_counter()
        x, si = op.solve(b, mg, tol, 100)
        torch.cuda.synchronize()
        w = time.perf_counter() - t
        best = w if best is None else min(best, w)
    z = torch.empty_like(b)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        mg.apply(b, z)
    e1.record()
    e1.synchronize()
    rel = float((b - op.apply(x)).norm() / b.norm())
    r.update(flag=si.flag, iters=si.iters, wall_s=round(best, 3), loop_ms=round(si.loop_ms, 1),
             vcycle_ms=round(e0.elapsed_time(e1) / 5, 3), true_relres=rel)
    del mg, z, x
    return r


def large(B, dev, mg_too, tol):
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, load_vector
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    free0 = _free(dev)
    r = {"block": B, "n": blk.n, "free_before_bytes": int(free0)}
    try:
        H = generate_box_operator(blk, device=dev)
        op = SubdomainOperator(H)
        b = load_vector(blk, device=dev)
        minv = op.jacobi()
        op.solve(b, minv, 0.0, 2, fixed_iters=True, check_every=2)
        _, info = op.solve(b, minv, 0.0, 20, fixed_iters=True, check_every=10, record_resvec=True)
        torch.cuda.synchronize()
        r.update(ok=True, ms_per_iter=round(info.loop_ms / 20, 3), free_drop_bytes=int(free0 - torch.cuda.mem_get_info(dev)[0]),
                 peak_torch_bytes=int(torch.cuda.max_memory_allocated(dev)), resvec_first_last=[float(info.resvec[0]), float(info.resvec[-1])])
        if mg_too:
            r["multigrid"] = large_mg(blk, op, b, minv, dev, tol)
        del op, H, b, minv
    except Exception as e:
        r.update(ok=False, error=str(e)[:300])
    _free(dev)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--contrast", type=float, default=100.0)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--large", type=str, default="512", help="comma-separated cube sizes for the large-box runs ('' = none)")
    ap.add_argument("--mg-large", action="store_true")
    ap.add_argument("--skip", type=str, default="", help="comma-separated sections to skip: compare,parity,mg")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hexop_bench: needs a CUDA device")
    from pcg_mpi_solver_b200.hexmesh import HexBlock, inclusion_field
    dev = torch.device("cuda:0")
    skip = set(s for s in a.skip.split(",") if s)
    B = a.block
    blk = HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B)
    out = {"block": B, "n": blk.n, "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats, **gpu_info()}
    if "compare" not in skip:
        out["uniform"] = compare(blk, dev, None, a)
        out["voxel"] = compare(blk, dev, inclusion_field(blk.ng, E_inclusion=a.contrast), a)
        out["voxel"]["contrast"] = a.contrast
    if "parity" not in skip:
        out["parity"] = parity(blk, dev, B)
    if "mg" not in skip:
        out["multigrid"] = multigrid(blk, dev, a.tol)
    sizes = [int(v) for v in a.large.split(",") if v]
    out["large"] = [large(v, dev, a.mg_large, a.tol) for v in sizes]
    print(json.dumps(out))
    if "parity" in out and not out["parity"]["ok"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
