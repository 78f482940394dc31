"""SpMV-only timing sweep over plan knobs (env PCGB_SPMV_*), 128^3 hex box.  Prints GB/s per config."""
import itertools, json, os, sys, time
sys.path.insert(0, ".")
import torch
from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_matrix
from pcg_mpi_solver_b200.csr import CsrMatrix
blk_n = int(os.environ.get("SWEEP_BLOCK", "128"))
dev = torch.device("cuda:0")
if os.environ.get("SWEEP_MODEL", "hex") == "concrete":
    # the irregular octree model (config C4, one part): 616 413 rows, 24..324 non-zeros per row
    from pcg_mpi_solver_b200.partition import assemble_csr_device, partition_mesh
    sub = partition_mesh(os.path.join("oracle", "_ref", "concrete.zip"), 1, assemble=False)[0]
    rp, col, val = assemble_csr_device(sub, dev)
    base = CsrMatrix(rp, col, val, (sub.n, sub.n))
else:
    blk = HexBlock((blk_n,) * 3, (0, 0, 0), (blk_n,) * 3, h=1.0 / blk_n)
    base = generate_matrix(blk, device=dev)
x = torch.randn(base.shape[1], dtype=torch.float64, device=dev)
y = torch.empty_like(x)
BSR = {"PCGB_SPMV_BSR": 1, "PCGB_SPMV_CTAS": 2, "PCGB_SPMV_STAGES": 2}
if os.environ.get("SWEEP_MODEL", "hex") == "concrete":
    default = [{"PCGB_SPMV_LANES": 16, "PCGB_SPMV_TILE": 1792, "PCGB_SPMV_STAGES": 4, "PCGB_SPMV_CTAS": 2}] + [
        {"PCGB_SPMV_LANES": l, "PCGB_SPMV_TILE": t, "PCGB_SPMV_STAGES": 2, "PCGB_SPMV_CTAS": 2} for l in (8, 16) for t in (2400, 2800, 3200, 3600)] + [
        {"PCGB_SPMV_LANES": 16, "PCGB_SPMV_TILE": 2000, "PCGB_SPMV_STAGES": 2, "PCGB_SPMV_CTAS": 3},
        {"PCGB_SPMV_LANES": 16, "PCGB_SPMV_TILE": 1280, "PCGB_SPMV_STAGES": 4, "PCGB_SPMV_CTAS": 3}]
else:
    default = [
        {"PCGB_SPMV_BSR": 0, "PCGB_SPMV_T3": 0, "PCGB_SPMV_LANES": 8, "PCGB_SPMV_TILE": 2304, "PCGB_SPMV_STAGES": 4, "PCGB_SPMV_CTAS": 2},      # round-1 kernel
        {"PCGB_SPMV_BSR": 1},                                            # library defaults: adaptive tile (largest with two CTAs per SM)
        *[{"PCGB_SPMV_CTAS": 1, "PCGB_SPMV_STAGES": 2, "PCGB_SPMV_TILE": t, "PCGB_BSR_CW": cw} for t in (9000, 11500) for cw in (8, 12)],
        {"PCGB_SPMV_CTAS": 1, "PCGB_SPMV_STAGES": 3, "PCGB_SPMV_TILE": 7600, "PCGB_BSR_CW": 12},
        {"PCGB_SPMV_CTAS": 1, "PCGB_SPMV_STAGES": 4, "PCGB_SPMV_TILE": 5800, "PCGB_BSR_CW": 12}]
configs = json.loads(os.environ.get("SWEEP_CONFIGS", "[]")) or default
for cfg in configs:
    for k in [k for k in os.environ if k.startswith("PCGB_")]:   # every config starts from the library defaults
        del os.environ[k]
    for k, v in cfg.items():
        os.environ[k] = str(v)
    M = CsrMatrix(base.rowptr, base.col, base.val, base.shape)
    for _ in range(3):
        M.spmv(x, out=y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        M.spmv(x, out=y)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print(json.dumps({**cfg, "ms": round(ms, 4), "GBps": round(M.spmv_bytes() / ms / 1e6, 1), "smem": M.plan_info()["smem_bytes"], "staged": M.plan_info()["staged"], "xcap": M.plan_info()["x_cap"], "maxw": M.plan_info()["max_windows_per_tile"], "mode": M.plan_info()["index_mode"], "lanes": M.plan_info()["lanes"],
                      "streamGBps": round(M.stream_bytes() / ms / 1e6, 1), "ctas": M.plan_info()["resident_ctas"],
                      "tile": M.plan_info()["tile_items"], "vdict": M.value_dict_blocks()}), flush=True)
    del M
