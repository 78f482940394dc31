"""Quick timing of the experimental EBE operator against the CSR kernel on the 128^3 hex box (1 GPU)."""
import gc, json, sys, time
sys.path.insert(0, ".")
import numpy as np, torch
from pcg_mpi_solver_b200.hexmesh import HexBlock, generate_ebe
from pcg_mpi_solver_b200.solver import SubdomainOperator
B = int(sys.argv[1]) if len(sys.argv) > 1 else 128
dev = torch.device("cuda:0")
t0 = time.time()
E = generate_ebe(HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B), device=dev)
op = SubdomainOperator(E)
n = E.shape[0]
x = torch.randn(n, dtype=torch.float64, device=dev); y = torch.empty_like(x)
for _ in range(3): E.apply_local(x, out=y)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20): E.apply_local(x, out=y)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 20
b = torch.zeros(n, dtype=torch.float64, device=dev); b[2::3] = -1e-4
minv = op.jacobi()
op.solve(b, minv, 0.0, 20, fixed_iters=True, check_every=20)
_, info = op.solve(b, minv, 0.0, 200, fixed_iters=True, check_every=50)
# coloured (atomics-free, bit-reproducible) variant of the same operator
from pcg_mpi_solver_b200.ebe import EbeMatrixColored
from pcg_mpi_solver_b200.hexmesh import hex_type_group
grp, eff, ndof = hex_type_group(HexBlock((B,) * 3, (0, 0, 0), (B,) * 3, h=1.0 / B))
C = EbeMatrixColored([grp], eff, ndof, device=dev)
yc = C.apply_local(x).clone()
for _ in range(3): C.apply_local(x)
torch.cuda.synchronize()
e0.record()
for _ in range(20): C.apply_local(x)
e1.record(); torch.cuda.synchronize()
ms_col = e0.elapsed_time(e1) / 20
yc2 = C.apply_local(x).clone()
colored = {"colored_apply_ms": ms_col, "colors": C.ncolors, "launches": C.launches()}
E.apply_local(x, out=y)
atomic = {"block": B, "n": n, "elements": B ** 3, "ebe_apply_ms": ms, "ebe_bytes": E.spmv_bytes(), "ebe_GBps": E.spmv_bytes() / ms / 1e6,
          "pcg_ms_per_iter": info.loop_ms / 200, "pcg_it_per_s": 200 / (info.loop_ms * 1e-3), "setup_s": time.time() - t0}
# the same coloured operator with every constant-memory slot taken by other pattern matrices: its 24-dof slices run on
# the warp kernel (Ke from global memory, the repeated-dof scan in the scatter)
from pcg_mpi_solver_b200.ebe import EbeMatrix
from pcg_mpi_solver_b200.partition import TypeGroup
del C, E, op
gc.collect()
rng = np.random.default_rng(0)
held = []
for _ in range(8):
    k = rng.standard_normal((24, 24))
    held.append(EbeMatrix([TypeGroup(0, np.arange(24)[:, None], np.zeros((24, 1), bool), np.ones(1), k + k.T, np.arange(1))],
                          np.arange(24), 24, device=dev))
Cw = EbeMatrixColored([grp], eff, ndof, device=dev)
ycw = Cw.apply_local(x).clone()
torch.cuda.synchronize()
e0.record()
for _ in range(20): Cw.apply_local(x)
e1.record(); torch.cuda.synchronize()
ms_warp = e0.elapsed_time(e1) / 20
colored_warp = {"colored_warp_apply_ms": ms_warp, "warp_launches": Cw.launches(), "warp_same_bits": bool(torch.equal(ycw, yc))}
del Cw, held
print(json.dumps({**colored, "colored_vs_atomic_max_rel_diff": float((yc - y).abs().max() / y.abs().max()),
                  "colored_bit_reproducible": bool(torch.equal(yc2, yc)), **colored_warp}))
print(json.dumps(atomic))
