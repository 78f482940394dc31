"""Effective-stiffness benchmark for periodic voxel cells (DESIGN §2.13).  For each size:
  apply     one application of the periodic index-free operator against k_hexop on the clamped box of the same element
            count (CUDA events, warm-up first), with algorithmic GB/s (pcgb_hexop_bytes: x and y once, the field once)
  average   one fused element pass and fixed-order average (pcgb_fields_average; bytes: x once, the field once)
  C_eff     effective_stiffness: Jacobi-PCG iterations and seconds per load case and the total, uniform (every case
            skipped: b is rounding noise) and inclusion_field (contrast 10)
Prints the card and its power limit (read in the same run), then one JSON line per case.  Needs a CUDA device."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.fields_bench import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--solve-sizes", type=int, nargs="*", default=None, help="sizes to run C_eff at (default: --sizes)")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--maxiter", type=int, default=20000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("homog_bench: needs a CUDA device")
    from pcg_mpi_solver_b200 import effective_stiffness
    from pcg_mpi_solver_b200.fields import PeriodicFields
    from pcg_mpi_solver_b200.hexmesh import HexBlock, PeriodicCell, generate_box_operator, generate_periodic_operator, inclusion_field
    dev = torch.device("cuda:0")
    name, limit = card()
    print(json.dumps({"card": name, "power_limit_and_max_sm_clock": limit}), flush=True)
    solve_sizes = args.sizes if args.solve_sizes is None else args.solve_sizes
    for n in sorted(set(args.sizes) | set(solve_sizes)):
        ne = (n, n, n)
        cell = PeriodicCell(ne, h=1.0 / n, nu=0.2)
        f = inclusion_field(ne, E_inclusion=10.0)
        if n in args.sizes:
            for kind, E_field in (("uniform", None), ("inclusion10", f)):
                op = generate_periodic_operator(cell, device=dev, E_field=E_field)
                x = torch.randn(cell.n, dtype=torch.float64, device=dev)
                y = torch.empty_like(x)
                ms = timed(lambda: op.apply_local(x, out=y), args.reps, args.warmup)
                blk = HexBlock(ne, (0, 0, 0), ne, h=1.0 / n, nu=0.2)
                box = generate_box_operator(blk, device=dev, E_field=E_field)
                xb = torch.randn(blk.n, dtype=torch.float64, device=dev)
                yb = torch.empty_like(xb)
                ms_box = timed(lambda: box.apply_local(xb, out=yb), args.reps, args.warmup)
                print(json.dumps({"case": "apply", "n": n, "field": kind, "periodic_ms": round(ms, 4), "box_ms": round(ms_box, 4),
                                  "periodic_GBps": round(op.spmv_bytes() / ms * 1e-6, 1),
                                  "box_GBps": round(box.spmv_bytes() / ms_box * 1e-6, 1)}), flush=True)
                del op, box, xb, yb
                F = PeriodicFields(cell, device=dev, E_field=E_field)
                strain = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0])
                ms = timed(lambda: F.average(x, strain), args.reps, args.warmup)
                nbytes = 8 * cell.n + (8 * cell.n_elements if E_field is not None else 0)
                print(json.dumps({"case": "average", "n": n, "field": kind, "ms": round(ms, 4),
                                  "GBps": round(nbytes / ms * 1e-6, 1)}), flush=True)
                del F, x, y
                torch.cuda.empty_cache()
        if n in solve_sizes:
            for kind, E_field in (("uniform", None), ("inclusion10", f)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                C, infos = effective_stiffness(cell, E_field=E_field, tol=args.tol, maxiter=args.maxiter, device=dev)
                torch.cuda.synchronize()
                total = time.perf_counter() - t0
                print(json.dumps({"case": "C_eff", "n": n, "field": kind, "tol": args.tol, "total_s": round(total, 3),
                                  "iters": [i.iters for i in infos], "flags": [i.flag for i in infos],
                                  "loop_s": [round(i.loop_ms * 1e-3, 3) for i in infos],
                                  "ms_per_iter": [round(i.loop_ms / i.iters, 3) if i.iters else None for i in infos],
                                  "C_diag": [float(C[k, k]) for k in range(6)],
                                  "asym": float(np.abs(C - C.T).max() / np.abs(C).max())}), flush=True)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
