"""Time to solution of Jacobi-PCG against multigrid-preconditioned PCG (HexMultigrid) on the bench's hex box.

    python tools/gmg_bench.py --block 128 --tol 1e-8 [--operator csr|ebe_ordered|ebe] [--repeats 3]
    python tools/gmg_bench.py --shape 200,150,75 --coarsening any

--shape NX,NY,NZ replaces the cubic --block box (h = 1 / NX); --coarsening any builds HexMultigrid(coarsening="any"), which
accepts any box.  Either option adds the level boxes, the Galerkin kernels' device time and the element-matrix peak of
`setup_info` to the multigrid line; without them the output is unchanged.

For each arm: iterations, flag, the device time of the loop (CUDA events inside the solve), the host wall time of the whole
solve (ending in a device synchronise), and for the multigrid arm its set-up time, the V-cycle time per application
(CUDA events around `pcgb_mg_apply`) and the hierarchy's device bytes next to the fine operator's: those the library
counts (vectors, coarse CSR, dense factor) and the drop in free device memory across the set-up, which also holds the coarse
SpMV plans' tables.  Prints one JSON line
per arm and the card's name, SM clock limit and power limit.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", type=int, default=128)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--operator", choices=["csr", "ebe_ordered", "ebe"], default="csr")
    ap.add_argument("--degree", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--vcycles", type=int, default=50)
    ap.add_argument("--coarsening", choices=["even", "any"], default="even")
    ap.add_argument("--shape", type=str, default=None, help="NX,NY,NZ (instead of --block)")
    a = ap.parse_args()
    shape = tuple(int(v) for v in a.shape.split(",")) if a.shape else (a.block,) * 3
    if len(shape) != 3 or min(shape) < 1:
        sys.exit("gmg_bench: --shape needs three positive element counts")
    extra = a.shape is not None or a.coarsening != "even"
    import torch
    if not torch.cuda.is_available():
        sys.exit("gmg_bench: needs a CUDA device")
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe, generate_matrix, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    dev = torch.device("cuda:0")
    B = a.block
    blk = HexBlock(shape, (0, 0, 0), shape, h=1.0 / shape[0])
    if a.operator == "csr":
        A = generate_matrix(blk, device=dev)
        op_bytes = A.val.numel() * 12 + A.rowptr.numel() * A.rowptr.element_size()
    else:
        A = generate_ebe(blk, device=dev, ordered=a.operator == "ebe_ordered")
        op_bytes = int(A.bytes()) if hasattr(A, "bytes") else None
    op = SubdomainOperator(A)
    b = load_vector(blk, device=dev)
    minv = op.jacobi()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0, _ = torch.cuda.mem_get_info(dev)
    t0 = time.perf_counter()
    mg = HexMultigrid(op, blk, degree=a.degree, minv=minv, coarsening=a.coarsening)
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t0
    free_drop = free0 - torch.cuda.mem_get_info(dev)[0]    # everything create took, the SpMV plans' tables included
    info = mg.info()

    def run(M, maxiter):
        op.solve(b, M, a.tol, maxiter)                         # warm-up (graph capture, module loads)
        best = None
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t = time.perf_counter()
            x, si = op.solve(b, M, a.tol, maxiter)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t
            if best is None or wall < best[0]:
                best = (wall, si, x)
        return best

    wj, ij, xj = run(minv, 20000)
    wm, im, xm = run(mg, 200)
    r = torch.empty_like(b)
    z = torch.empty_like(b)
    r.copy_(b)
    mg.apply(r, z)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.vcycles):
        mg.apply(r, z)
    e1.record()
    e1.synchronize()
    vc_ms = e0.elapsed_time(e1) / a.vcycles
    diff = float((xm - xj).norm() / xj.norm())
    common = {"block": B, "operator": a.operator, "tol": a.tol, "card": card()}
    if extra:
        common = {"shape": list(shape), "coarsening": a.coarsening, "operator": a.operator, "tol": a.tol, "card": card()}
    print(json.dumps({**common, "arm": "jacobi", "flag": ij.flag, "iters": ij.iters, "loop_ms": round(ij.loop_ms, 3),
                      "wall_s": round(wj, 4), "ms_per_iter": round(ij.loop_ms / max(ij.loop_iters, 1), 4)}))
    print(json.dumps({**common, "arm": "multigrid", "flag": im.flag, "iters": im.iters, "loop_ms": round(im.loop_ms, 3),
                      "wall_s": round(wm, 4), "ms_per_iter": round(im.loop_ms / max(im.loop_iters, 1), 4),
                      "vcycle_ms": round(vc_ms, 4), "setup_s": round(setup_s, 3), "degree": a.degree, "levels": info["levels"],
                      "n_levels": info["n"], "lambda": [round(v, 4) for v in info["lambda"]], "hierarchy_bytes": info["bytes"], "device_free_drop_bytes": free_drop,
                      "fine_operator_bytes": op_bytes, "speedup_wall": round(wj / wm, 2),
                      "x_rel_diff_vs_jacobi": diff,
                      **({"level_shapes": [list(v) for v in mg.level_shapes()], **mg.setup_info()} if extra else {})}))


if __name__ == "__main__":
    main()
