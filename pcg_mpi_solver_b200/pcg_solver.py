"""File-format-compatible solver stage: a drop-in for `mpiexec -np N python3 src/solver/pcg_solver.py RunId SpeedTestFlag`.

    python -m pcg_mpi_solver_b200.pcg_solver <RunId> <SpeedTestFlag>                                   # 1 part, 1 GPU
    python -m torch.distributed.run --nproc-per-node N -m pcg_mpi_solver_b200.pcg_solver <RunId> <SpeedTestFlag>

Reads exactly what the reference's solver reads (cwd-relative, pcg_solver.py:56,93-106,116):
    __pycache__/ModelDataPaths.zpkl, __pycache__/GlobSettings.zpkl,
    <PyDataPath_Part><N>_metadat.npy and <N>_<rank>.mpidat        (written by the reference's partition_mesh.py
                                                                   or by export_mesh_parts() below)
and writes what it writes (pcg_solver.py:142-209, 841-896, 943-961; file_operations.py:348-375):
    <Scratch>/Results_Run<R>/ResVecData/{Dof,NodeId,U_<k>}.mpidat + *_metadat.npy + Time_T.npy
    <Scratch>/Results_Run<R>/PlotData/<Model>_MP<N>_TimeData.{npz,mat}   (Flag / Iter / RelRes per load step, timers)
so that `src/data/export_vtk.py` keeps working unchanged.  The time-step shell (pcg_solver.py:1002-1008:
updateBC -> updatePreconditioner -> PCG -> export, same A and M for every load step) is kept as thin host code.
Displacement `U` is the only export variable supported: reference-format parts carry no strain modes, so the `PS`/`PE`
exports of pcg_solver.py:879-889 cannot run on them.  For hex boxes and voxel models, `fields.HexFields` recovers element
strains and stresses, principal values and their nodal averages on the device (DESIGN §2.10).
"""
from __future__ import annotations

import os
import pickle
import sys
import zlib
from datetime import datetime
from time import time

import numpy as np


# ------------------------------------------------------------------------------- small file helpers
def importz(path):
    """file_operations.py:38-42"""
    with open(path, "rb") as f:
        return pickle.loads(zlib.decompress(f.read()))


def exportz(path, data):
    """file_operations.py:32-36"""
    with open(path, "wb") as f:
        f.write(zlib.compress(pickle.dumps(data, pickle.HIGHEST_PROTOCOL)))


def read_mesh_part(prefix: str, nparts: int, rank: int) -> dict:
    """readModelData, pcg_solver.py:100-106: `<prefix><N>_<rank>.mpidat` = zlib(pickle(RefMeshPart))."""
    base = prefix + str(nparts)
    meta = np.load(base + "_metadat.npy", allow_pickle=True).item()
    raw = np.fromfile(f"{base}_{rank}.mpidat", dtype=meta["DTypeData"][rank], count=meta["NfData"][rank])
    return pickle.loads(zlib.decompress(raw.tobytes()))


def export_mesh_parts(prefix: str, subs, glob_extra=None):
    """Write SubdomainData parts in the reference's fixture format (exportMP, partition_mesh.py:1303-1369), with
    the keys the solver stage reads.  Lets the whole pipeline run without the reference's builder."""
    nparts = len(subs)
    bufs = []
    for s in subs:
        mp_ = s.to_refmeshpart()
        mp_["NodeWeightVector"] = mp_["DofWeightVector"][0::3].copy()
        # keys the reference's OWN solver stage reads besides the hot-path ones (pcg_solver.py:144-148, 365, 901-902)
        mp_["RefPlotData"] = {"TestPlotFlag": False, "J": [], "LocalDofVec": [], "DofVec": np.zeros(0, dtype=int), "RefPlotDofVec": [], "qpoint": []}
        mp_["MPList_RefPlotDofIndicesList"] = []
        mp_["GlobData"].update(glob_extra or {})
        mp_["GlobData"].setdefault("dt", 0.0)
        bufs.append(np.frombuffer(zlib.compress(pickle.dumps(mp_, pickle.HIGHEST_PROTOCOL)), "b"))
    os.makedirs(os.path.dirname(prefix), exist_ok=True)
    mem = np.array([b.nbytes for b in bufs])
    meta = np.array({"NfData": np.array([len(b) for b in bufs], dtype=object), "DTypeData": np.array([b.dtype for b in bufs], dtype=object),
                     "OffsetData": np.cumsum(np.hstack([[0], mem[:-1]]))}, dtype=object)
    np.save(prefix + str(nparts) + "_metadat", meta)
    for i, b in enumerate(bufs):
        b.tofile(f"{prefix}{nparts}_{i}.mpidat")


class _Ranks:
    """Minimal rank context: torch.distributed when launched with torchrun, else a single rank."""

    def __init__(self):
        self.rank = int(os.environ.get("RANK", "0"))
        self.size = int(os.environ.get("WORLD_SIZE", "1"))
        self.dist = None
        if self.size > 1:
            import torch
            import torch.distributed as dist
            backend = os.environ.get("PCGB_DIST_BACKEND", "nccl")   # "gloo": CPU tests of the multi-rank host logic
            if backend == "nccl":
                torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", self.rank)))
            if not dist.is_initialized():
                dist.init_process_group(backend)
            self.dist = dist

    def gather(self, obj):
        if self.size == 1:
            return [obj]
        out = [None] * self.size
        self.dist.all_gather_object(out, obj)
        return out

    def barrier(self):
        if self.size > 1:
            self.dist.barrier()


def write_mpi_file(path: str, data: np.ndarray, ranks: _Ranks):
    """writeMPIFile_parallel (file_operations.py:348-375): every rank writes its buffer at the gathered offset
    into `<path>.mpidat`; rank 0 writes `<path>_metadat.npy` {NfData, DTypeData, OffsetData}."""
    data = np.ascontiguousarray(data)
    metas = ranks.gather([data.nbytes, len(data), data.dtype])
    mem = np.array([m[0] for m in metas])
    offsets = np.cumsum(np.hstack([[0], mem[:-1]]))
    if ranks.rank == 0:
        meta = np.array({"NfData": np.array([m[1] for m in metas], dtype=object), "DTypeData": np.array([m[2] for m in metas], dtype=object),
                         "OffsetData": offsets}, dtype=object)
        np.save(path + "_metadat", meta)
        open(path + ".mpidat", "ab").close()
    ranks.barrier()
    fd = os.open(path + ".mpidat", os.O_WRONLY | os.O_CREAT, 0o644)
    os.pwrite(fd, data.tobytes(), int(offsets[ranks.rank]))
    os.close(fd)
    ranks.barrier()


# ------------------------------------------------------------------------------- the solver stage
def _default_backend(mp, ranks):
    """CUDA backend: assemble K[Eff,Eff] on this rank's GPU, NCCL communicator when there are several parts."""
    import torch
    from .partition import SubdomainData, TypeGroup
    from .solver import Communicator
    eff = np.asarray(mp["LocDofEff"], dtype=np.int64)
    groups = [TypeGroup(int(g["ElemTypeId"]), np.asarray(g["ElemList_LocDofVector"]), np.asarray(g["ElemList_SignVector"], dtype=bool),
                        np.asarray(g["ElemList_Ck"], dtype=float), np.asarray(g["ElemStiffMat"], dtype=float), None)
              for g in mp["SubDomainData"]["StrucDataList"] if int(g["ElemTypeId"]) >= 0]
    is_eff = np.zeros(mp["NDOF"], dtype=bool)
    is_eff[eff] = True
    pos = np.cumsum(is_eff) - 1
    ovrlp_full = [np.asarray(d, dtype=np.int64) for d in mp["OvrlpLocalDofVecList"]]
    ovrlp = [pos[d[is_eff[d]]] for d in ovrlp_full]
    sub = SubdomainData(int(mp["Id"]), ranks.size, np.asarray(mp["DofVector"]), np.asarray(mp["NodeIdVector"]), eff, groups,
                        [int(v) for v in mp["NbrMPIdVector"]], ovrlp_full, ovrlp, np.asarray(mp["DofWeightVector"], dtype=float),
                        np.asarray(mp["RefLoadVector"], dtype=float), np.asarray(mp["Ud"], dtype=float),
                        int(mp["GlobData"]["GlobNDofEff"]), int(mp["GlobData"]["GlobNDof"]))
    dev = torch.device(f"cuda:{torch.cuda.current_device()}")
    comm = Communicator.from_torch_distributed(dev) if ranks.size > 1 else None
    op = sub.to_operator(comm, device=dev)
    minv = op.jacobi()                                        # updatePreconditioner (:346-352): A does not change between steps

    def solve_step(b_eff, x0_eff, tol, maxiter):
        x, info = op.solve(torch.from_numpy(b_eff).to(dev), minv, tol, maxiter, x0=torch.from_numpy(x0_eff).to(dev))
        if info.too_small_tol:
            raise Warning("PCG : TooSmallTolerance")         # pcg_solver.py:549
        return x.cpu().numpy(), info.flag, info.relres, info.iters

    return sub, solve_step


def run(run_id, speed_test: int = 0, workdir: str = ".", backend=None, quiet: bool = False):
    """The `__main__` of the reference's pcg_solver.py (:965-1031) for this rank.  `backend(mp, ranks)` returns
    (SubdomainData, solve_step); the default runs on the GPU (tests inject a CPU checker to exercise the file formats)."""
    ranks = _Ranks()
    t_begin = time()
    paths = importz(os.path.join(workdir, "__pycache__", "ModelDataPaths.zpkl"))       # initGlobData :56-60
    settings = importz(os.path.join(workdir, "__pycache__", "GlobSettings.zpkl"))      # readGlobalSettings :116-132
    th, sp = settings["TimeHistoryParam"], settings["SolverParam"]
    res_path = paths["ScratchPath"] + "/Results_Run" + str(run_id) + ("_SpeedTest/" if speed_test == 1 else "/")
    plot_path, vec_path = res_path + "PlotData/", res_path + "ResVecData/"
    if ranks.rank == 0:
        if os.path.exists(res_path):
            os.rename(res_path, res_path[:-1] + "_" + datetime.now().strftime("%d%m%Y_%H%M%S"))   # :68-70
        os.makedirs(plot_path)
        os.makedirs(vec_path)
        if not quiet:
            print(">loading partitioned data..")
    ranks.barrier()
    mp = read_mesh_part(paths["PyDataPath_Part"], ranks.size, ranks.rank)
    t_read = time() - t_begin
    export_flag = bool(th["ExportFlag"]) and speed_test != 1 and "U" in th["ExportVars"]
    deltas = list(th["TimeStepDelta"])
    nsteps = len(deltas)
    dt = float(mp["GlobData"].get("dt", 0.0))
    sub, solve_step = (backend or _default_backend)(mp, ranks)
    eff = sub.loc_dof_eff
    t_start = time()
    if ranks.rank == 0 and not quiet:
        print(f">running parallel pcg solver with {ranks.size} GPUs..")
    un = np.zeros(sub.ndof)                                            # :996 (1e-200*rand: numerically zero)
    own_dof = sub.weights_full.astype(bool)
    own_node = own_dof[0::3]
    export_count = 0
    times_t = []
    # ExportFrms is a nested 1-based list in the reference: np.array(ExportFrms, int)[0] - 1  (initExportData, :156-159)
    frms = np.array(th["ExportFrms"], dtype=int)
    frms = (frms[0] - 1) if len(frms) > 0 else frms
    frms = set(int(v) for v in np.atleast_1d(frms))
    rate = th["ExportFrmRate"]

    def export_now(step):                                              # exportContourData :854-859
        return (rate > 0 and step % rate == 0) or (step in frms)

    def export_frame(step):
        nonlocal export_count
        write_mpi_file(vec_path + "U_" + str(export_count), un[own_dof], ranks)   # :867-869
        times_t.append(step * dt)                                      # TimeList[TimeStepCount] = TimeStepCount*dt (:167)
        if ranks.rank == 0:
            np.save(vec_path + "Time_T", times_t)
        export_count += 1

    if export_flag:                                                    # initExportData :195-209 (calls exportContourData at step 0)
        write_mpi_file(vec_path + "Dof", sub.dof_vector[own_dof], ranks)
        write_mpi_file(vec_path + "NodeId", sub.node_ids[own_node], ranks)
        if export_now(0):
            export_frame(0)
    flags, relres, iters = np.zeros(nsteps), np.zeros(nsteps), np.zeros(nsteps)
    from .partition import _ebe_matvec
    for step in range(1, nsteps):                                      # :1002-1008
        delta = deltas[step]
        udi = sub.Ud * delta                                           # updateBC :234-238
        fdi = np.zeros(sub.ndof)
        if any(ranks.gather(bool(np.any(udi != 0)))):                  # K (Ud delta) + the interface sum of calcMPFint (:303-334):
            fdi = _ebe_matvec(sub.groups, udi, sub.ndof)               # only the overlap dofs travel, neighbour by neighbour
            sends = ranks.gather({q: fdi[idx] for q, idx in zip(sub.nbr, sub.ovrlp_full)})
            recv = [sends[q][ranks.rank] for q in sub.nbr]
            for idx, vals in zip(sub.ovrlp_full, recv):                # += in neighbour order (:332-334)
                fdi[idx] += vals
        fext = sub.F * delta - fdi
        x, flag, rr, it = solve_step(fext[eff], un[eff], sp["Tol"], sp["MaxIter"])
        if it > 0 or flag != 0:
            flags[step], relres[step], iters[step] = flag, rr, it      # :593-596
            xunq = np.zeros(sub.ndof)
            xunq[eff] = x
            un = xunq + udi                                            # :598
        # else: PCG returned early (zero right-hand side or initial guess good enough, :387-395, :421-426): the reference's
        # early `return` leaves RefMeshPart['Un'] and the TimeList_* entries untouched
        if export_flag and export_now(step):
            export_frame(step)
    t_end = time()
    rec = ranks.gather({"dT_FileRead": t_read, "dT_Calc": t_end - t_start, "dT_CommWait": 0.0, "t0_Start": t_start, "t0_End": t_end})
    if ranks.rank == 0:                                                # exportTimeData :943-961 / configTimeRecData
        ts0, te1 = min(r["t0_Start"] for r in rec), max(r["t0_End"] for r in rec)
        wait = np.array([(r["t0_Start"] - ts0) + (te1 - r["t0_End"]) for r in rec])
        time_data = {"TotalTime": te1 - ts0, "MaxCommWaitTime": float(wait.max()), "MinCommWaitTime": float(wait.min()),
                     "Mean_FileReadTime": float(np.mean([r["dT_FileRead"] for r in rec])),
                     "Mean_CalcTime": float(np.mean([r["dT_Calc"] for r in rec])), "Mean_CommWaitTime": float(wait.mean()),
                     "Max_TotalTime_i": float(max(r["dT_Calc"] for r in rec)), "LoadUnbalanceData": [], "PBS_JobId": 0,
                     "Flag": flags, "Iter": iters, "RelRes": relres}
        name = plot_path + paths["ModelName"] + "_MP" + str(ranks.size) + "_TimeData"
        np.savez_compressed(name, TimeData=time_data)
        try:
            from scipy.io import savemat
            savemat(name + ".mat", time_data)
        except Exception:
            pass
        if not quiet:
            print(">success!")
            print(f"\n>file read time:     {np.round(time_data['Mean_FileReadTime'], 1)} sec \n>calculation time:   {np.round(time_data['Mean_CalcTime'], 1)} sec\n"
                  f">communication time: {np.round(time_data['Mean_CommWaitTime'], 1)} sec\n>---------------------------\n"
                  f">total runtime:      {np.round(time_data['TotalTime'], 1)} sec \n")
    ranks.barrier()
    return {"Flag": flags, "Iter": iters, "RelRes": relres, "Un": un, "sub": sub}


if __name__ == "__main__":
    run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 0)
