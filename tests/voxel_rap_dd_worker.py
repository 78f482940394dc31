"""Multi-rank worker for the rap voxel multigrid across ranks (launched by tests/test_gpu_voxel_rap_dd.py through
torch.distributed.run; argv: out.json split combos, split "grid:PX,PY,PZ:PER" or "tile:NX,NY,NZ:W0,W1,..." (x widths),
combos "kind:contrast,..." with kind csr or box).

For every combo every rank draws the same global inclusion_field (contrast 1: a constant field), builds its operator from
its block_field slice and three hierarchies: HexMultigrid(coarse="rap") and the ranked field hierarchy (coarse="csr") on
the same boxes, and the one-rank rap handle of the global mesh.  Checks, per rank:
- levels, shapes and gather level equal to the ranked field hierarchy's; level 1's D^-1, every ranked and replicated level
  >= 2 (CSR, D^-1, lambda) and the coarsest solve torch.equal / == to it;
- level 1's local product (level_apply) within 1e-13 of each row's |A||x| of the field hierarchy's level-1 CSR times x;
- the exchange-added level-1 product: rows of nodes no other rank holds bit-identical to the one-rank rap product, the
  others within 1e-14 (max-relative); the ranked lambda within 1e-12 of the one-rank lambda;
- the V-cycle within 1e-12 (normwise) of the one-rank rap handle's and of the field hierarchy's; shared copies of z equal to
  1e-13 across ranks;
- MG-PCG to 1e-8 in the iteration count of the one-rank rap handle and of the field hierarchy, x within 1e-9 of the one-rank
  x; launches per iteration the same over two windows and on every rank;
- a repeated set-up bit-identical; info()["bytes"] == rap_rank_bytes;
- refusals (a NaN in the last rank's part of the field; at the C entry n_ranked = 1 and a NaN Ck) on every rank alike,
  allocating nothing.
Split "large" runs 2x1x1 ranks of 256^3 (index-free fine operator, contrast 10) against the one-rank rap handle of the
512x256x256 mesh, built once on rank 0: equal iterations, x within 1e-9, and the device-wide drop in free memory across the
ranks' second set-up within 2 % of the sum of rap_rank_bytes and the ranks' fields (the SpMV and halo plans are not counted).
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
import scipy.sparse as sp
import torch
import torch.distributed as dist


def main():
    out_path, split = sys.argv[1], sys.argv[2]
    combos = [(c.split(":")[0], float(c.split(":")[1])) for c in sys.argv[3].split(",")] if len(sys.argv) > 3 else []
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    timeout = datetime.timedelta(seconds=600)
    if shared:
        dist.init_process_group("gloo", timeout=timeout)
    else:
        dist.init_process_group("nccl", device_id=dev, timeout=timeout)
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import (HexBlock, block_field, generate_box_operator, generate_matrix, inclusion_field,
                                             interface_lists, load_vector, partition_blocks)
    from pcg_mpi_solver_b200.multigrid import HexMultigrid, rank_levels, rap_rank_bytes
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator, make_halo
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    lib = _lib.load()
    fails, stats = [], []
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

    kind_s, a, b_ = (split.split(":") + ["", ""])[:3]
    if kind_s == "grid":
        pgrid, per = tuple(int(v) for v in a.split(",")), int(b_)
        ng = tuple(pgrid[i] * per for i in range(3))
        blocks = [HexBlock(b.ng, b.e0, b.ne, h=1.0 / ng[0]) for b in partition_blocks(ng, pgrid)]
    elif kind_s == "tile":
        ng, widths = tuple(int(v) for v in a.split(",")), [int(v) for v in b_.split(",")]
        blocks, x = [], 0
        for w in widths:
            blocks.append(HexBlock(ng, (x, 0, 0), (w, ng[1], ng[2]), h=1.0 / ng[0]))
            x += w
    else:                                                   # "large"
        ng = (512, 256, 256)
        blocks = [HexBlock(b.ng, b.e0, b.ne, h=1.0 / ng[0]) for b in partition_blocks(ng, (2, 1, 1))]
        combos = [("box", 10.0)]
    assert len(blocks) == world
    h = 1.0 / ng[0]
    blk = blocks[rank]
    levels = rank_levels(blocks)
    la_want = len(levels) - 1
    gblk = HexBlock(ng, (0, 0, 0), ng, h=h)
    n_global = 3 * ng[0] * (ng[1] + 1) * (ng[2] + 1)
    nbr, lists, w = interface_lists(blocks, rank)

    def gmap(b):
        lz, ly, lx = np.meshgrid(np.arange(b.ne[2] + 1), np.arange(b.ne[1] + 1), np.arange(b.x_lo, b.ne[0] + 1), indexing="ij")
        gn = ((lz.ravel() + b.e0[2]) * (b.ng[1] + 1) + ly.ravel() + b.e0[1]) * b.ng[0] + (lx.ravel() + b.e0[0] - 1)
        return (3 * gn[:, None] + np.arange(3)[None, :]).ravel()

    maps = [gmap(lv[rank]) for lv in levels]

    def alone(fn):
        """Ranks sharing one GPU see one device-wide free-memory figure: each runs fn in its own turn, the others waiting."""
        torch.cuda.synchronize()
        dist.barrier()
        for turn in range(world):
            if turn == rank:
                fn()
            dist.barrier()

    if kind_s == "large":
        large(locals())
        combos = []

    for kind, contrast in combos:
        st = {"kind": kind, "contrast": contrast}
        field = inclusion_field(ng, 0.4, (1.0, max(2.0, ng[1] / 8)), 1.0, contrast, seed=29)
        fb = block_field(field, blk)
        A = generate_matrix(blk, device=dev, E_field=fb) if kind == "csr" else generate_box_operator(blk, device=dev, E_field=fb)
        op = SubdomainOperator(A, comm, nbr, lists, w, n_global=n_global)
        mg = HexMultigrid(op, blk, blocks=blocks, E_field=field, coarse="rap")
        fh = HexMultigrid(op, blk, blocks=blocks, E_field=field)
        op1 = SubdomainOperator(generate_matrix(gblk, device=dev, E_field=field))
        mg1 = HexMultigrid(op1, gblk, E_field=field, coarse="rap")
        info, infof, info1 = mg.info(), fh.info(), mg1.info()
        la, nlev = info["gather_level"], info["levels"]
        st.update(levels=nlev, gather_level=la, bytes=info["bytes"], bytes_field=infof["bytes"], setup=mg.setup_info(),
                  setup_field=fh.setup_info())
        note(la == la_want and la == infof["gather_level"] and info["n"] == infof["n"], "levels differ from the field hierarchy")
        note(mg.level_shapes() == fh.level_shapes(), "level shapes differ from the field hierarchy")
        note(nlev - 1 == info1["levels"], f"levels {nlev} vs one-rank {info1['levels']}")
        note(info["bytes"] == rap_rank_bytes(levels, rank), f"bytes {info['bytes']} vs rap_rank_bytes {rap_rank_bytes(levels, rank)}")

        # level 1's D^-1 and every level >= 2: the ranked field hierarchy's bit for bit
        note(torch.equal(mg.level_dinv(1), fh.level_dinv(1)), "level-1 D^-1 differs from the field hierarchy's")
        for k in range(2, nlev - 1):
            if k == la:
                continue
            note(all(torch.equal(x, y) for x, y in zip(mg.level_matrix(k), fh.level_matrix(k))), f"level {k} CSR differs")
            note(torch.equal(mg.level_dinv(k), fh.level_dinv(k)), f"level {k} D^-1 differs")
            note(info["lambda"][k] == infof["lambda"][k], f"level {k} lambda {info['lambda'][k]} vs {infof['lambda'][k]}")
        rng = np.random.default_rng(1234)             # the same draws on every rank
        rc = t(rng.standard_normal(info["n"][-1]))
        note(torch.equal(mg.coarse_solve(rc), fh.coarse_solve(rc)), "coarsest solve differs")

        # level 1's local product against the field hierarchy's level-1 CSR
        rp, col, val = (v.cpu().numpy() for v in fh.level_matrix(1))
        A1 = sp.csr_matrix((val, col, rp), shape=(info["n"][1],) * 2)
        x1 = rng.standard_normal(info1["n"][1])
        xl = x1[maps[1]]
        y = mg.level_apply(1, t(xl)).cpu().numpy()
        bound = abs(A1) @ np.abs(xl)
        loc = float(np.max(np.abs(y - A1 @ xl) / bound))
        note(loc <= 1e-13, f"level-1 local product off the field CSR by {loc:.3e} of |A||x|")
        # the exchange-added product against the one-rank rap handle
        yt = t(y)
        _lib.check(lib.pcgb_halo_exchange_add(mg._halos[0], _lib.ptr(yt), _lib.stream_ptr()), "pcgb_halo_exchange_add")
        ya = yt.cpu().numpy()
        y1 = mg1.level_apply(1, t(x1)).cpu().numpy()[maps[1]]
        _, lists1, _ = interface_lists(levels[1], rank)
        shared_dof = np.zeros(maps[1].size, dtype=bool)
        for li in lists1:
            shared_dof[li] = True
        inner = ~shared_dof
        bad = int(np.sum(ya[inner].view(np.uint64) != y1[inner].view(np.uint64)))
        note(bad == 0, f"level 1: {bad} interior rows differ from the one-rank rap product")
        iface = float(np.max(np.abs(ya[shared_dof] - y1[shared_dof]), initial=0.0) / np.max(np.abs(y1)))
        note(iface <= 1e-14, f"level 1: interface rows off the one-rank product by {iface:.3e}")
        lam = abs(info["global_lambda"][1] - info1["lambda"][1]) / info1["lambda"][1]
        note(lam <= 1e-12, f"ranked lambda_1 off the one-rank lambda by {lam:.3e}")
        st.update(local_rel=loc, interior_rows=int(inner.sum()), interface_rel=iface, lambda1_rel=lam)

        # the V-cycle
        r = rng.standard_normal(n_global)
        zt = mg.apply(t(r[maps[0]]))
        z = zt.cpu().numpy()
        want = mg1.apply(t(r)).cpu().numpy()[maps[0]]
        zf = fh.apply(t(r[maps[0]])).cpu().numpy()
        e1 = float(np.linalg.norm(z - want) / np.linalg.norm(want))
        ef = float(np.linalg.norm(z - zf) / np.linalg.norm(zf))
        note(e1 <= 1e-12, f"V-cycle off the one-rank rap V-cycle by {e1:.3e}")
        note(ef <= 1e-12, f"V-cycle off the field hierarchy's by {ef:.3e}")
        zg = np.full(n_global, np.nan)
        spread = 0.0
        for mm, v in allg((maps[0], z)):
            seen = ~np.isnan(zg[mm])
            spread = max(spread, float(np.max(np.abs(zg[mm][seen] - v[seen]), initial=0.0)))
            zg[mm] = v
        note(spread <= 1e-13 * np.abs(want).max(), f"shared copies of z differ by {spread:.3e}")
        st.update(vcycle_vs_one_rank=e1, vcycle_vs_field=ef, z_copy_spread=spread / np.abs(want).max())

        # MG-PCG
        b = load_vector(blk, device=dev)
        x, si = op.solve(b, mg, 1e-8, 300)
        _, sf = op.solve(b, fh, 1e-8, 300)
        x1s, s1 = op1.solve(load_vector(gblk, device=dev), mg1, 1e-8, 300)
        xe = float((x - x1s[torch.from_numpy(maps[0]).to(dev)]).norm() / x1s.norm())
        note(si.flag == 0 and si.iters == s1.iters == sf.iters, f"MG-PCG iters {si.iters} vs one-rank {s1.iters}, field {sf.iters}")
        note(xe <= 1e-9, f"x off the one-rank x by {xe:.3e}")
        ls = []
        for maxiter in (6, 12, 18):
            _, ii = op.solve(b, mg, 1e-30, maxiter, fixed_iters=True, check_every=6)
            ls.append(ii.launches)
        per6 = [ls[1] - ls[0], ls[2] - ls[1]]
        note(per6[0] == per6[1], f"launches per 6 iterations not constant: {per6}")
        note(len({tuple(p) for p in allg(per6)}) == 1, f"launches per 6 iterations differ across ranks: {per6}")
        st.update(iters=si.iters, iters_one_rank=s1.iters, iters_field=sf.iters, x_vs_one_rank=xe, launches_per_6=per6[0])

        # a repeated set-up is bit-identical
        mg2 = HexMultigrid(op, blk, blocks=blocks, E_field=field, coarse="rap")
        same = [float(v).hex() for v in mg2.info()["lambda"]] == [float(v).hex() for v in info["lambda"]]
        same = same and all(torch.equal(mg.level_dinv(k), mg2.level_dinv(k)) for k in range(1, nlev - 1) if k != la)
        for k in range(2, nlev - 1):
            if k != la:
                same = same and all(torch.equal(p, q) for p, q in zip(mg.level_matrix(k), mg2.level_matrix(k)))
        same = same and torch.equal(mg2.apply(t(r[maps[0]])), zt)
        note(same, "a repeated set-up differs")
        del mg2
        stats.append(st)

        # refusals: the same on every rank, nothing allocated
        if contrast == combos[-1][1] and kind == combos[-1][0]:
            stats[-1]["refusals"] = refusals(locals())
        del mg, fh, mg1, op, op1, A
        gc.collect()
        torch.cuda.synchronize()

    torch.cuda.synchronize()
    status = lib.pcgb_comm_status(comm.handle, _lib.stream_ptr())
    note(status == 0, f"communicator status {status}")
    xs = allg((fails, stats, time.time() - t0))
    if rank == 0:
        res = {"world": world, "split": split, "transport": comm.transport, "fails": [f for g_ in xs for f in g_[0]],
               "stats": [g_[1] for g_ in xs], "seconds": max(g_[2] for g_ in xs)}
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


def refusals(env) -> int:
    """A NaN in the last rank's part of the global field (HexMultigrid), and at the C entry n_ranked = 1 and a NaN Ck."""
    import torch.distributed as dist  # noqa: F401
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.hexmesh import interface_lists
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import make_halo
    op, blk, blocks, field, fh, levels, ng = (env[k] for k in ("op", "blk", "blocks", "field", "fh", "levels", "ng"))
    rank, world, dev, comm, lib, note, alone = (env[k] for k in ("rank", "world", "dev", "comm", "lib", "note", "alone"))
    gc.collect()
    torch.cuda.synchronize()
    count = [0]
    fnan = field.copy()
    fnan[ng[2] - 1, ng[1] - 1, ng[0] - 1] = float("nan")         # in the last rank's box

    def python_refusal():
        free0 = torch.cuda.mem_get_info(dev)[0]
        try:
            HexMultigrid(op, blk, blocks=blocks, E_field=fnan, coarse="rap")
            note(False, "NaN in the global field: accepted")
        except ValueError:
            count[0] += 1
        torch.cuda.synchronize()
        note(torch.cuda.mem_get_info(dev)[0] >= free0, "the Python refusal allocated device memory")

    alone(python_refusal)
    la = len(levels) - 1
    g = levels[la][0].ng
    nke = 576 * g[0] * g[1] * g[2]
    others = [q for q in range(world) if q != rank]
    kg = make_halo(comm, others, [np.arange(nke, dtype=np.int64)] * len(others), nke)
    ck = torch.full((blk.ne[0] * blk.ne[1] * blk.ne[2],), blk.h, dtype=torch.float64, device=dev)
    minv = op.jacobi()
    halos = (ctypes.c_void_p * la)(*[hh.value for hh in fh._halos[:la]])
    own = [torch.from_numpy(interface_lists(lv, rank)[2]).to(dev) for lv in levels]
    owns = (ctypes.c_void_p * (la + 1))(*[o.data_ptr() for o in own])
    ke = np.ascontiguousarray(np.eye(24))
    box = blk.cbox()
    torch.cuda.synchronize()

    def c_refusal(n_ranked, what):
        out = ctypes.c_void_p()
        free0 = torch.cuda.mem_get_info(dev)[0]
        rc = lib.pcgb_mg_create_ranks_field_rap(op._solver, ctypes.byref(box), n_ranked, halos, fh._gather, kg, owns,
                                                ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _lib.ptr(ck), _lib.ptr(minv),
                                                2, 0.25, ctypes.byref(out))
        torch.cuda.synchronize()
        note(rc == -1 and not out, f"pcgb_mg_create_ranks_field_rap with {what}: rc {rc}")
        note(torch.cuda.mem_get_info(dev)[0] >= free0, f"the C refusal ({what}) allocated device memory")
        count[0] += rc == -1

    alone(lambda: c_refusal(1, "n_ranked = 1"))
    ck[3] = float("nan")
    torch.cuda.synchronize()
    alone(lambda: c_refusal(la, "a NaN Ck"))
    lib.pcgb_halo_destroy(kg)
    return count[0]


def large(env):
    """2x1x1 ranks of 256^3 against the one-rank rap handle of 512x256x256, built once on rank 0."""
    from pcg_mpi_solver_b200.hexmesh import block_field, generate_box_operator, inclusion_field, load_vector
    from pcg_mpi_solver_b200.multigrid import HexMultigrid, rap_rank_bytes
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    rank, world, dev, comm, blocks, blk, ng, gblk, levels, maps, note, allg, stats = (
        env[k] for k in ("rank", "world", "dev", "comm", "blocks", "blk", "ng", "gblk", "levels", "maps", "note", "allg", "stats"))
    nbr, lists, w, n_global = env["nbr"], env["lists"], env["w"], env["n_global"]
    st = {"kind": "box", "contrast": 10.0, "large": True}
    free = torch.cuda.mem_get_info(dev)[0]
    if min(allg(free)) < 60e9:
        st["skipped"] = f"{free / 1e9:.1f} GB free"
        stats.append(st)
        return
    field = inclusion_field(ng, 0.4, (2.0, 6.0), 1.0, 10.0, seed=29)
    op = SubdomainOperator(generate_box_operator(blk, device=dev, E_field=block_field(field, blk)), comm, nbr, lists, w,
                           n_global=n_global)
    minv = op.jacobi()
    b = load_vector(blk, device=dev)
    predicted = sum(rap_rank_bytes(levels, r) + 8 * bb.ne[0] * bb.ne[1] * bb.ne[2] for r, bb in enumerate(blocks))

    def build():
        """A set-up and the device-wide drop in free memory across it (both ranks' set-ups)."""
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        dist.barrier()
        free0 = torch.cuda.mem_get_info(dev)[0]
        dist.barrier()
        t0 = time.perf_counter()
        M = HexMultigrid(op, blk, minv=minv, blocks=blocks, E_field=field, coarse="rap")
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        torch.cuda.empty_cache()
        dist.barrier()
        d = free0 - torch.cuda.mem_get_info(dev)[0]
        dist.barrier()
        return M, dt, d

    # The first set-up of the process also grows the driver's and the caching allocator's pools for its many small
    # allocations (halo plans, SpMV plans, the coarse levels' vectors), which stay after it is destroyed; the second set-up's
    # drop is the hierarchy's own.
    mg, _, drop_first = build()
    del mg
    gc.collect()
    mg, setup_s, drop = build()
    # info()["bytes"], like rap_bytes, leaves out the SpMV plans of the CSR levels (2-byte indices per 3x3 block, tile
    # descriptors) and the halo plans; at 256^3 per rank, where level 2's CSR is a fifth of the hierarchy, they add 1.4 %
    rel = abs(drop - predicted) / predicted
    note(rel <= 0.02, f"free-memory drop {drop} vs predicted {predicted} ({rel:.3%}; first set-up {drop_first})")
    note(mg.info()["bytes"] == rap_rank_bytes(levels, rank), "bytes differ from rap_rank_bytes")
    x, si = op.solve(b, mg, 1e-8, 300)
    st.update(setup_s=round(setup_s, 3), bytes=mg.info()["bytes"], setup=mg.setup_info(), free_drop_both_ranks=int(drop), first_free_drop_both_ranks=int(drop_first),
              predicted_both_ranks=int(predicted), drop_rel=rel, iters=si.iters)
    xl = x.cpu().numpy()
    del mg, op, x
    gc.collect()
    torch.cuda.empty_cache()
    dist.barrier()
    tmp = os.path.dirname(os.path.abspath(env["out_path"]))
    if rank == 0:                                  # the one-rank handle, built once
        op1 = SubdomainOperator(generate_box_operator(gblk, device=dev, E_field=field))
        mg1 = HexMultigrid(op1, gblk, E_field=field, coarse="rap")
        x1, s1 = op1.solve(load_vector(gblk, device=dev), mg1, 1e-8, 300)
        x1 = x1.cpu().numpy()
        for r in range(world):
            np.save(os.path.join(tmp, f"x1_{r}.npy"), x1[env["gmap"](levels[0][r])])
        st1 = [s1.iters, float(np.linalg.norm(x1))]
        del mg1, op1
        gc.collect()
        torch.cuda.empty_cache()
    else:
        st1 = None
    dist.barrier()
    it1, n1 = [s for s in allg(st1) if s is not None][0]
    x1 = np.load(os.path.join(tmp, f"x1_{rank}.npy"))
    xe = float(np.linalg.norm(xl - x1) / n1)
    note(si.flag == 0 and si.iters == it1, f"large: MG-PCG iters {si.iters} vs one-rank {it1}")
    note(xe <= 1e-9, f"large: x off the one-rank x by {xe:.3e}")
    st.update(iters_one_rank=it1, x_vs_one_rank=xe)
    stats.append(st)


if __name__ == "__main__":
    main()
