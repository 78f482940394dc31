"""Timing of the field recovery (csrc/fields.cuh, HexFields) on cubic hex boxes, uniform and with an inclusion_field:
the element pass with all four outputs and with stress only, the nodal average of the principal stresses, and one
application of the index-free operator (hexop) on the same box for scale.

    python tools/fields_bench.py [--sizes 128 256 512] [--reps 20] [--warmup 3] [--uniform-only]

x is a deterministic smooth field computed on the device (no solve).  Each entry is timed with CUDA events around `reps`
calls after `warmup` calls, outputs preallocated, through the C ABI.  Bytes are algorithmic, from the shapes:
  element   x once (8 per free dof) + the field (8 per element) + the outputs (8 per component per element)
  nodal     the element pass into scratch (x, field, 24 per element written), the nodal sum (24 per element read, 32 per
            node written) and the division (32 per node read, 24 written)
  hexop     pcgb_hexop_bytes (x and y once, the field once)
Prints the card and its power limit (read in the same run), then one JSON line per case.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK_BW = 3.35e12   # H100 SXM data-sheet HBM3 bandwidth


def smooth_x(blk, dev):
    nx, ny, nz = blk.ne
    lx = torch.arange(blk.x_lo, nx + 1, device=dev, dtype=torch.float64) / nx
    ly = torch.arange(ny + 1, device=dev, dtype=torch.float64) / ny
    lz = torch.arange(nz + 1, device=dev, dtype=torch.float64) / nz
    Z, Y, X = torch.meshgrid(lz, ly, lx, indexing="ij")
    u = torch.empty(Z.shape + (3,), dtype=torch.float64, device=dev)
    u[..., 0] = torch.sin(1.3 * X + 0.7 * Y) * (1.0 + Z)
    u[..., 1] = 0.4 * X * X - torch.cos(2.1 * Z + Y)
    u[..., 2] = X * Y * Z + 0.25 * torch.sin(3.0 * Y)
    del X, Y, Z
    return (u.reshape(-1) * 1e-3).contiguous()


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the name is still printed; the limit is reported missing, not guessed
        q = f"unavailable ({e})"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[128, 256, 512])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--uniform-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fields_bench: needs a CUDA device")
    from pcg_mpi_solver_b200 import HexFields, _lib
    from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_box_operator, inclusion_field
    dev = torch.device("cuda:0")
    name, limit = card()
    print(json.dumps({"card": name, "power_limit_and_max_sm_clock": limit}), flush=True)
    lib = _lib.load()
    st = lambda: _lib.stream_ptr()   # noqa: E731
    for n in args.sizes:
        for field in ([False] if args.uniform_only else [False, True]):
            blk = HexBlock((n, n, n), (0, 0, 0), (n, n, n), h=1.0 / n)
            f = torch.from_numpy(inclusion_field(blk.ne, seed=0)).to(dev) if field else None
            ne, nn = n ** 3, (n + 1) ** 3
            x = smooth_x(blk, dev)
            F = HexFields(blk, device=dev, E_field=f)
            rows = []
            fb = 8 * ne if field else 0
            o6a, o6b, o3a, o3b = (torch.empty(ne * k, dtype=torch.float64, device=dev) for k in (6, 6, 3, 3))
            h = F._h
            ms = timed(lambda: _lib.check(lib.pcgb_fields_element(h, _lib.ptr(x), _lib.ptr(o6a), _lib.ptr(o6b), _lib.ptr(o3a),
                                                                  _lib.ptr(o3b), st())), args.reps, args.warmup)
            rows.append(("element_all", ms, 8 * blk.n + fb + 8 * 18 * ne))
            ms = timed(lambda: _lib.check(lib.pcgb_fields_element(h, _lib.ptr(x), None, _lib.ptr(o6b), None, None, st())),
                       args.reps, args.warmup)
            rows.append(("element_stress", ms, 8 * blk.n + fb + 8 * 6 * ne))
            del o6a, o6b, o3a, o3b
            work = torch.empty(4 * nn, dtype=torch.float64, device=dev)
            out = torch.empty(3 * nn, dtype=torch.float64, device=dev)
            ms = timed(lambda: _lib.check(lib.pcgb_fields_nodal(h, _lib.ptr(x), 0, None, _lib.ptr(work), _lib.ptr(out), st())),
                       args.reps, args.warmup)
            rows.append(("nodal_stress", ms, 8 * blk.n + fb + 24 * ne + 24 * ne + 32 * nn + 32 * nn + 24 * nn))
            ok = bool(torch.isfinite(out).all().item())
            del work, out
            op = generate_box_operator(blk, device=dev, E_field=f)
            y = torch.empty_like(x)
            ms = timed(lambda: op.apply_local(x, out=y), args.reps, args.warmup)
            rows.append(("hexop_apply", ms, op.spmv_bytes()))
            del op, y, F, x, f
            torch.cuda.empty_cache()
            for what, ms, by in rows:
                gbs = by / (ms * 1e-3) / 1e9
                print(json.dumps({"n": n, "field": field, "case": what, "ms": round(ms, 4), "bytes": int(by), "GB_s": round(gbs, 1),
                                  "share_of_3.35TB_s": round(gbs * 1e9 / PEAK_BW, 3), "nodal_finite": ok}), flush=True)


if __name__ == "__main__":
    main()
