"""Multi-rank worker for the voxel-model multigrid across ranks (launched by tests/test_gpu_voxel_mg_dd.py through
torch.distributed.run; argv: out.json pgrid per kind contrast).

Every rank draws the same global inclusion_field (contrast 1: a constant field), cuts its box out with block_field,
builds its operator (csr / ebe_ordered / box) and HexMultigrid(op, block, blocks=..., E_field=global field).  It also
builds the uniform ranked handle on the same boxes and the one-rank field hierarchy of the global mesh on its own.  Checks,
per rank:
- levels, level shapes and gather level equal to the uniform ranked handle's;
- every replicated level's CSR torch.equal to the one-rank level of the same global level, and its lambda equal;
- ranked levels: rows of nodes no other rank holds bit-identical to the one-rank rows, the exchange-added A_l x within
  1e-14 (max-relative) of the one-rank product, lambda within 1e-12 of the one-rank lambda;
- the V-cycle within 1e-12 (normwise) of the one-rank handle's, shared copies of z equal to 1e-13 across ranks;
- contrast 1: the V-cycle within 1e-11 of the uniform ranked handle's (one-rank field against one-rank uniform recorded);
- MG-PCG to 1e-8 in the one-rank field MG-PCG's iteration count, fewer than half of Jacobi-PCG's on the same split, x
  within 1e-9 of the one-rank x;
- launches per PCG iteration equal to the uniform ranked handle's;
- a repeated set-up bit-identical (level CSRs, lambda, V-cycle);
- refusals (NaN in the global field, the rank's block-shaped field, index-free, coarsening="any", a NaN Ck at the C entry
  point) raised on every rank alike, allocating nothing.
Ranks never raise on a mismatch: they record it, and rank 0 writes every rank's findings."""
import ctypes
import datetime
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist


def main():
    out_path, pgrid, per, kind = sys.argv[1], tuple(int(v) for v in sys.argv[2].split(",")), int(sys.argv[3]), sys.argv[4]
    contrast = float(sys.argv[5])
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    timeout = datetime.timedelta(seconds=300)
    if shared:
        dist.init_process_group("gloo", timeout=timeout)
    else:
        dist.init_process_group("nccl", device_id=dev, timeout=timeout)
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import (HexBlock, block_field, generate_box_operator, generate_ebe, generate_matrix,
                                             inclusion_field, interface_lists, load_vector, partition_blocks)
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator, make_halo
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    lib = _lib.load()
    fails, stats = [], {}
    t0 = time.time()

    def allg(obj):
        box = [None] * world
        dist.all_gather_object(box, obj)
        return box

    def t(v):
        return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)

    def note(ok, what):
        if not ok:
            fails.append(f"rank {rank} {what}")

    ng = tuple(pgrid[a] * per for a in range(3))
    h = 1.0 / ng[0]
    blocks = [HexBlock(b.ng, b.e0, b.ne, h=h) for b in partition_blocks(ng, pgrid)]
    blk = blocks[rank]
    field = inclusion_field(ng, 0.4, (1.0, per / 3), 1.0, contrast, seed=23)
    fb = block_field(field, blk)

    def operator(b, f):
        if kind == "csr":
            return generate_matrix(b, device=dev, E_field=f)
        if kind == "ebe_ordered":
            return generate_ebe(b, device=dev, ordered=True, E_field=f)
        return generate_box_operator(b, device=dev, E_field=f)

    nbr, lists, w = interface_lists(blocks, rank)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    op = SubdomainOperator(operator(blk, fb), comm, nbr, lists, w, n_global=n_global)
    mg = HexMultigrid(op, blk, blocks=blocks, E_field=field)
    uni = HexMultigrid(op, blk, blocks=blocks)
    info, infou = mg.info(), uni.info()
    la = info["gather_level"]
    nlev = info["levels"]
    gblk = HexBlock(ng, (0, 0, 0), ng, h=h)
    op1 = SubdomainOperator(generate_matrix(gblk, device=dev, E_field=field))
    mg1 = HexMultigrid(op1, gblk, E_field=field)
    info1 = mg1.info()
    stats.update(levels=nlev, gather_level=la, n_gathered=info["n_gathered"], setup=mg.setup_info())
    note(nlev == infou["levels"] and la == infou["gather_level"] and info["n"] == infou["n"], "levels / sizes differ from the uniform handle")
    note(mg.level_shapes() == uni.level_shapes(), "level shapes differ from the uniform handle")
    note(nlev - 1 == info1["levels"], f"levels {nlev} vs one-rank {info1['levels']}")

    # replicated levels: the one-rank field levels la, la + 1, ... bit for bit
    for k in range(la + 1, nlev - 1):
        a, b = mg.level_matrix(k), mg1.level_matrix(k - 1)
        note(all(torch.equal(x, y) for x, y in zip(a, b)), f"replicated level {k} CSR differs from one-rank level {k - 1}")
        note(info["lambda"][k] == info1["lambda"][k - 1], f"replicated level {k} lambda {info['lambda'][k]} vs {info1['lambda'][k - 1]}")
    glam = info["global_lambda"]
    lam_err = max([abs(a - b) / b for a, b in zip(glam[:la], info1["lambda"][:la])], default=0.0)
    stats["lambda_rel_err"] = lam_err
    note(lam_err <= 1e-12, f"ranked lambda off the one-rank lambda by {lam_err:.3e}")

    # per-level boxes and global dof maps (hexmesh numbering, global box x = 0 clamped)
    def half(b):
        return HexBlock(tuple(v // 2 for v in b.ng), tuple(v // 2 for v in b.e0), tuple(v // 2 for v in b.ne), h=2 * b.h)

    lvl = [blocks]
    for _ in range(la):
        lvl.append([half(b) for b in lvl[-1]])

    def gmap(b):
        lz, ly, lx = np.meshgrid(np.arange(b.ne[2] + 1), np.arange(b.ne[1] + 1), np.arange(b.x_lo, b.ne[0] + 1), indexing="ij")
        gn = ((lz.ravel() + b.e0[2]) * (b.ng[1] + 1) + ly.ravel() + b.e0[1]) * b.ng[0] + (lx.ravel() + b.e0[0] - 1)
        return (3 * gn[:, None] + np.arange(3)[None, :]).ravel()

    maps = [gmap(lv[rank]) for lv in lvl]
    rng = np.random.default_rng(1234)            # the same draws on every rank
    interior_rows, worst_ax = 0, 0.0
    for l in range(1, la):
        rp, col, val = (v.cpu().numpy() for v in mg.level_matrix(l))
        rp1, col1, val1 = (v.cpu().numpy() for v in mg1.level_matrix(l))
        m = maps[l]
        _, lists_l, _ = interface_lists(lvl[l], rank)
        shared_dof = np.zeros(m.size, dtype=bool)
        for li in lists_l:
            shared_dof[li] = True
        bad = 0
        for i in np.flatnonzero(~shared_dof):
            g = m[i]
            c, v = m[col[rp[i]:rp[i + 1]]], val[rp[i]:rp[i + 1]]
            c1, v1 = col1[rp1[g]:rp1[g + 1]], val1[rp1[g]:rp1[g + 1]]
            if not (np.array_equal(c, c1) and np.array_equal(v.view(np.uint64), v1.view(np.uint64))):
                bad += 1
        interior_rows += int(np.sum(~shared_dof))
        note(bad == 0, f"ranked level {l}: {bad} interior rows differ from the one-rank rows")
        x = rng.standard_normal(info1["n"][l])
        y = mg.level_apply(l, t(x[m]))
        _lib.check(lib.pcgb_halo_exchange_add(mg._halos[l - 1], _lib.ptr(y), _lib.stream_ptr()), "pcgb_halo_exchange_add")
        y1 = mg1.level_apply(l, t(x)).cpu().numpy()
        err = float(np.max(np.abs(y.cpu().numpy() - y1[m])) / np.max(np.abs(y1)))
        worst_ax = max(worst_ax, err)
    stats.update(interior_rows=interior_rows, ax_rel_err=worst_ax)
    note(worst_ax <= 1e-14, f"exchange-added A_l x off the one-rank product by {worst_ax:.3e}")

    # the whole V-cycle against the one-rank handle's
    r = rng.standard_normal(n_global)
    zt = mg.apply(t(r[maps[0]]))
    z = zt.cpu().numpy()
    want = mg1.apply(t(r)).cpu().numpy()[maps[0]]
    err = float(np.linalg.norm(z - want) / np.linalg.norm(want))
    stats["vcycle_rel_err"] = err
    note(err <= 1e-12, f"V-cycle off the one-rank V-cycle by {err:.3e}")
    allz = allg((maps[0], z))
    zg = np.full(n_global, np.nan)
    spread = 0.0
    for mm, v in allz:
        seen = ~np.isnan(zg[mm])
        spread = max(spread, float(np.max(np.abs(zg[mm][seen] - v[seen]), initial=0.0)))
        zg[mm] = v
    stats["z_copy_spread"] = spread / np.abs(want).max()
    note(spread <= 1e-13 * np.abs(want).max(), f"shared copies of z differ by {spread:.3e}")
    if contrast == 1.0:
        # Galerkin products and rediscretisations of a constant field differ by rounding, which the V-cycle amplifies
        # with the box's aspect: the same comparison on one rank is recorded beside it (DESIGN 2.9)
        zu = uni.apply(t(r[maps[0]])).cpu().numpy()
        eu = float(np.linalg.norm(z - zu) / np.linalg.norm(zu))
        zu1 = HexMultigrid(op1, gblk).apply(t(r)).cpu().numpy()[maps[0]]
        stats["vcycle_vs_uniform"] = eu
        stats["vcycle_vs_uniform_one_rank"] = float(np.linalg.norm(want - zu1) / np.linalg.norm(zu1))
        note(eu <= 1e-11, f"constant field: V-cycle off the uniform ranked handle's by {eu:.3e}")

    # MG-PCG
    b = load_vector(blk, device=dev)
    x, si = op.solve(b, mg, 1e-8, 300)
    bg = load_vector(gblk, device=dev)
    x1, s1 = op1.solve(bg, mg1, 1e-8, 300)
    _, sj = op.solve(b, op.jacobi(), 1e-8, 50000)
    xe = float((x - x1[torch.from_numpy(maps[0]).to(dev)]).norm() / x1.norm())
    stats.update(iters=si.iters, iters_one_rank=s1.iters, iters_jacobi=sj.iters, x_vs_one_rank=xe)
    note(si.flag == 0 and si.iters == s1.iters, f"MG-PCG flag {si.flag} iters {si.iters} vs one-rank {s1.iters}")
    note(sj.flag == 0 and 2 * si.iters < sj.iters, f"MG-PCG {si.iters} iterations vs Jacobi {sj.iters}")
    note(xe <= 1e-9, f"x off the one-rank x by {xe:.3e}")
    per_it = []
    for M in (mg, uni):
        ls = []
        for maxiter in (6, 12):
            _, ii = op.solve(b, M, 1e-30, maxiter, fixed_iters=True, check_every=6)
            ls.append(ii.launches)
        per_it.append(ls[1] - ls[0])
    stats["launches_per_6_iters"] = per_it
    note(per_it[0] == per_it[1], f"launches per 6 iterations {per_it[0]} vs uniform {per_it[1]}")

    # a repeated set-up is bit-identical
    mg2 = HexMultigrid(op, blk, blocks=blocks, E_field=field)
    same = [float(v).hex() for v in mg2.info()["lambda"]] == [float(v).hex() for v in info["lambda"]]
    for k in range(1, nlev - 1):
        if k != la:
            same = same and all(torch.equal(a, c) for a, c in zip(mg.level_matrix(k), mg2.level_matrix(k)))
    same = same and torch.equal(mg2.apply(t(r[maps[0]])), zt)
    note(same, "a repeated set-up differs")
    del mg2

    # refusals: the same on every rank, nothing allocated.  Ranks sharing one GPU see one device-wide free-memory figure, so
    # each rank measures its refusals in its own turn while the others wait at a barrier, their work finished.
    def alone(fn):
        torch.cuda.synchronize()
        dist.barrier()
        for turn in range(world):
            if turn == rank:
                fn()
            dist.barrier()

    gc.collect()
    torch.cuda.synchronize()
    refusals = 0
    fnan = field.copy()
    fnan[ng[2] - 1, ng[1] - 1, ng[0] - 1] = float("nan")         # in the last rank's box

    def python_refusals():
        nonlocal refusals
        free0 = torch.cuda.mem_get_info(dev)[0]
        for what, kw in (("NaN in the global field", dict(E_field=fnan)), ("block-shaped field", dict(E_field=fb)),
                         ("index_free", dict(E_field=field, coarse="index_free")), ("any", dict(E_field=field, coarsening="any"))):
            try:
                HexMultigrid(op, blk, blocks=blocks, **kw)
                fails.append(f"rank {rank} refusal {what}: accepted")
            except ValueError:
                refusals += 1
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info(dev)[0]
        note(free1 >= free0, f"a refusal allocated device memory ({free0 - free1} bytes)")

    alone(python_refusals)
    # the C entry point: a NaN Ck on every rank, with a valid element plan
    g = lvl[la][0].ng
    nke = 576 * g[0] * g[1] * g[2]
    others = [q for q in range(world) if q != rank]
    kg = make_halo(comm, others, [np.arange(nke, dtype=np.int64)] * len(others), nke)
    ck = torch.full((blk.ne[0] * blk.ne[1] * blk.ne[2],), h, dtype=torch.float64, device=dev)
    ck[3] = float("nan")
    minv = op.jacobi()
    halos = (ctypes.c_void_p * la)(*[hh.value for hh in uni._halos[:la]])
    own = [torch.from_numpy(interface_lists(lv, rank)[2]).to(dev) for lv in lvl]
    owns = (ctypes.c_void_p * (la + 1))(*[o.data_ptr() for o in own])
    ke = np.ascontiguousarray(np.eye(24))
    box = blk.cbox()
    torch.cuda.synchronize()

    def c_refusal():
        nonlocal refusals
        out = ctypes.c_void_p()
        free0 = torch.cuda.mem_get_info(dev)[0]
        rc = lib.pcgb_mg_create_ranks_field(op._solver, ctypes.byref(box), la, halos, uni._gather, kg, owns,
                                            ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _lib.ptr(ck), _lib.ptr(minv), 2, 0.25,
                                            ctypes.byref(out))
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info(dev)[0]
        note(rc == -1 and not out, f"pcgb_mg_create_ranks_field with a NaN Ck: rc {rc}")
        note(free1 >= free0, f"the C refusal allocated device memory ({free0 - free1} bytes)")
        refusals += rc == -1

    alone(c_refusal)
    lib.pcgb_halo_destroy(kg)
    stats["refusals"] = refusals

    torch.cuda.synchronize()
    status = lib.pcgb_comm_status(comm.handle, _lib.stream_ptr())
    note(status == 0, f"communicator status {status}")
    xs = allg((fails, stats, time.time() - t0))
    if rank == 0:
        res = {"world": world, "pgrid": list(pgrid), "per": per, "kind": kind, "contrast": contrast, "transport": comm.transport,
               "fails": [f for g_ in xs for f in g_[0]], "stats": [g_[1] for g_ in xs], "seconds": max(g_[2] for g_ in xs)}
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
