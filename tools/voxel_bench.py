"""Time to solution of Jacobi-PCG against multigrid-preconditioned PCG on a voxel model: a hex box with one Young's modulus
per element (hexmesh.inclusion_field: spherical inclusions of E_matrix * contrast in a matrix of E_matrix = 1).

    python tools/voxel_bench.py --block 128 --contrast 10 [--fraction 0.4] [--operator csr|ebe_ordered|ebe|hexop]
                                [--coarse csr|rap] [--jacobi-fixed N] [--repeats 3]

For each arm one JSON line: iterations, flag, the device time of the loop (CUDA events inside the solve) and the host wall
time of the whole solve (ending in a device synchronise).  The multigrid arm adds its set-up wall time, the device time of
its Galerkin kernels, the hierarchy's device bytes as the library counts them, the drop in free device memory across the
set-up, the peak bytes of element matrices held during it, and the value-dictionary size of the fine matrix (CSR operator)
and of every coarse level (0: more distinct 3x3 blocks than the dictionary holds, the plain node-block kernel).  Every line
carries the card's name, power limit and SM clock.  Needs a GPU; there is no CPU path.

--coarse rap builds the multigrid with a matrix-free level 1 (HexMultigrid(coarse="rap")), the one whose hierarchy fits a
512^3 voxel model on one GPU (with --operator hexop).  --jacobi-fixed N replaces the Jacobi solve by N fixed iterations and
reports their ms per iteration (a full Jacobi solve at 512^3 takes minutes).  A third line ("arm": "level1") times one
level-1 application three ways in the same process: the fused P^T A_0 P kernel of a rap hierarchy, the three launches it
fuses (prolongation into a zero fine vector, the index-free fine operator of the field, restriction), and the CSR
level-1 SpMV of the CSR field hierarchy when that hierarchy fits (null otherwise); the hierarchy the arm did not build is
built for this line after the solves.
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", type=int, default=128)
    ap.add_argument("--contrast", type=float, default=10.0)
    ap.add_argument("--fraction", type=float, default=0.4)
    ap.add_argument("--radii", type=float, nargs=2, default=(2.0, 6.0))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--operator", choices=["csr", "ebe_ordered", "ebe", "hexop"], default="csr")
    ap.add_argument("--coarse", choices=["csr", "rap"], default="csr")
    ap.add_argument("--jacobi-fixed", type=int, default=0, help="time N fixed Jacobi iterations instead of a full solve")
    ap.add_argument("--level1-reps", type=int, default=20)
    ap.add_argument("--degree", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--jacobi-maxiter", type=int, default=50000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("voxel_bench: needs a CUDA device")
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, generate_ebe, generate_matrix, inclusion_field, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid, rap_bytes
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    dev = torch.device("cuda:0")
    B = a.block
    blk = HexBlock((B, B, B), (0, 0, 0), (B, B, B), h=1.0 / B)
    field = inclusion_field(blk.ng, a.fraction, tuple(a.radii), 1.0, a.contrast, a.seed)
    if a.operator == "csr":
        A = generate_matrix(blk, device=dev, E_field=field)
        fine_dict = A.value_dict_blocks()
    elif a.operator == "hexop":
        A = generate_box_operator(blk, device=dev, E_field=field)
        fine_dict = None
    else:
        A = generate_ebe(blk, device=dev, ordered=a.operator == "ebe_ordered", E_field=field)
        fine_dict = None
    op = SubdomainOperator(A)
    b = load_vector(blk, device=dev)
    minv = op.jacobi()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0, _ = torch.cuda.mem_get_info(dev)
    t0 = time.perf_counter()
    mg = HexMultigrid(op, blk, degree=a.degree, minv=minv, E_field=field, coarse=a.coarse)
    torch.cuda.synchronize()
    setup_s = time.perf_counter() - t0
    free_drop = free0 - torch.cuda.mem_get_info(dev)[0]
    info, sinfo = mg.info(), mg.setup_info()
    level_dict = []
    for l in range(1, info["levels"] - 1):
        if a.coarse == "rap" and l == 1:    # matrix-free
            level_dict.append(None)
            continue
        rp, col, val = mg.level_matrix(l)
        M = CsrMatrix(rp, col, val, (info["n"][l], info["n"][l]))
        level_dict.append(M.value_dict_blocks())
        del M, rp, col, val
    torch.cuda.empty_cache()

    def run(M, maxiter):
        op.solve(b, M, a.tol, maxiter)                          # warm-up (graph capture, module loads)
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

    if a.jacobi_fixed:
        op.solve(b, minv, a.tol, a.jacobi_fixed, fixed_iters=True)
        torch.cuda.synchronize()
        t = time.perf_counter()
        xj, ij = op.solve(b, minv, a.tol, a.jacobi_fixed, fixed_iters=True)
        torch.cuda.synchronize()
        wj = time.perf_counter() - t
    else:
        wj, ij, xj = run(minv, a.jacobi_maxiter)
    wm, im, xm = run(mg, 1000)
    common = {"block": B, "operator": a.operator, "contrast": a.contrast, "fraction": a.fraction,
              "inclusion_fraction": round(float((field != 1.0).mean()), 4), "tol": a.tol, "card": card()}
    jline = {**common, "arm": "jacobi", "flag": ij.flag, "iters": ij.iters, "loop_ms": round(ij.loop_ms, 3),
             "wall_s": round(wj, 4), "ms_per_iter": round(ij.loop_ms / max(ij.loop_iters, 1), 4), "fine_value_dict_blocks": fine_dict}
    if a.jacobi_fixed:
        jline["fixed_iters"] = a.jacobi_fixed
    print(json.dumps(jline))
    mline_extra = {} if a.coarse == "csr" else {"coarse": a.coarse, "rap_bytes": rap_bytes(blk.ne)}
    print(json.dumps({**common, "arm": "multigrid", "flag": im.flag, "iters": im.iters, "loop_ms": round(im.loop_ms, 3),
                      "wall_s": round(wm, 4), "ms_per_iter": round(im.loop_ms / max(im.loop_iters, 1), 4),
                      "setup_s": round(setup_s, 3), "galerkin_ms": round(sinfo["galerkin_ms"], 3),
                      "element_matrix_peak_bytes": sinfo["element_matrix_peak_bytes"], "degree": a.degree,
                      "levels": info["levels"], "n_levels": info["n"], "lambda": [round(v, 4) for v in info["lambda"]],
                      "hierarchy_bytes": info["bytes"], "device_free_drop_bytes": free_drop,
                      "fine_value_dict_blocks": fine_dict, "level_value_dict_blocks": level_dict,
                      "speedup_wall": round(wj / wm, 2), "speedup_wall_with_setup": round(wj / (wm + setup_s), 2),
                      "x_rel_diff_vs_jacobi": None if a.jacobi_fixed else float((xm - xj).norm() / xj.norm()), **mline_extra}))
    del xj, xm
    print(json.dumps({**common, "arm": "level1", **level1_times(a, dev, blk, field, op, A, mg, minv)}))


def level1_times(a, dev, blk, field, op, A, mg, minv):
    """ms of one level-1 application, each over a.level1_reps back-to-back launches between CUDA events after one warm-up:
    the fused kernel (rap), the three launches it fuses, and the CSR field hierarchy's level-1 SpMV where it fits."""
    import torch
    from pcg_mpi_solver_b200.hexop import HexBoxOperator
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    csr_fits = blk.ne[0] * blk.ne[1] * blk.ne[2] <= 256 ** 3
    if a.coarse == "rap":
        mr, mc = mg, (HexMultigrid(op, blk, degree=a.degree, minv=minv, E_field=field) if csr_fits else None)
    else:
        mr, mc = HexMultigrid(op, blk, degree=a.degree, minv=minv, E_field=field, coarse="rap"), mg
    A0 = A if a.operator == "hexop" else HexBoxOperator(blk, device=dev, E_field=field)
    n1 = mr.info()["n"][1]
    x = torch.randn(n1, dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    y = torch.empty_like(x)
    u = torch.zeros(op.n, dtype=torch.float64, device=dev)
    v = torch.empty_like(u)

    def composed():
        u.zero_()
        mr.prolong_add(0, x, u)
        A0.apply_local(u, out=v)
        return mr.restrict(0, v)

    def timed(fn):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.level1_reps):
            fn()
        e1.record()
        e1.synchronize()
        return round(e0.elapsed_time(e1) / a.level1_reps, 4)

    out = {"n_level1": n1, "reps": a.level1_reps, "fused_ms": timed(lambda: mr.level_apply(1, x, out=y)),
           "composed_ms": timed(composed), "csr_spmv_ms": timed(lambda: mc.level_apply(1, x, out=y)) if mc is not None else None}
    out["fused_equals_composed"] = bool(torch.equal(mr.level_apply(1, x), composed()))
    return out


if __name__ == "__main__":
    main()
