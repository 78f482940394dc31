"""Multi-rank worker for the field recovery (launched by tests/test_gpu_fields_dd.py through torch.distributed.run; argv:
out.json field).

Every rank owns one box of partition_blocks(ng, block_grid(world)) and recovers its fields from the global mesh's smooth
displacement (fields_cases.smooth_x) restricted to its box, with HexFields(..., comm, blocks) (node-level halo plan).  It
also runs HexFields on the whole mesh as one box and compares its own part: element fields and the nodal values at nodes
no other rank holds bit for bit, and at interface nodes the counts exactly and the values to 8 ulp of the node's largest
value.  Ranks never raise on a mismatch: they record it, and rank 0 writes every rank's findings."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist


def _bits(a, b):
    return bool(np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64)))


def _raw(F, x, kind):
    """(work, out) of pcgb_fields_nodal with the object's halo plan."""
    from pcg_mpi_solver_b200 import _lib
    work = torch.empty((F.n_nodes, 4), dtype=torch.float64, device=F.device)
    out = torch.empty((F.n_nodes, 3), dtype=torch.float64, device=F.device)
    _lib.check(_lib.load().pcgb_fields_nodal(F._h, _lib.ptr(x), kind, F._halo, _lib.ptr(work), _lib.ptr(out), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return work.cpu().numpy(), out.cpu().numpy()


def main():
    out_path, field = sys.argv[1], sys.argv[2] == "1"
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    dist.init_process_group("gloo")
    from pcg_mpi_solver_b200 import HexFields
    from pcg_mpi_solver_b200.hexmesh import HexBlock, block_field, block_grid, interface_node_lists, partition_blocks
    from pcg_mpi_solver_b200.solver import Communicator
    from tests import fields_cases as C
    comm = Communicator.from_torch_distributed(dev, nccl=False)
    ng = (13, 10, 7)
    blocks = partition_blocks(ng, block_grid(world))
    for b_ in blocks:
        b_.h, b_.nu = 1.0 / ng[0], 0.27
    blk = blocks[rank]
    G = HexBlock(ng, (0, 0, 0), ng, h=1.0 / ng[0], nu=0.27)
    gfield = np.random.default_rng(11).uniform(0.1, 10.0, tuple(reversed(ng))) if field else None
    gx = C.smooth_x(G)
    x = torch.from_numpy(C.restrict_x(G, gx, blk)).to(dev)
    F = HexFields(blk, device=dev, E_field=block_field(gfield, blk) if field else None, comm=comm, blocks=blocks)
    Fg = HexFields(G, device=dev, E_field=gfield)
    xg = torch.from_numpy(gx).to(dev)
    el, elg = F.element(x), Fg.element(xg)
    ge, gn = C.global_elements(blk), C.global_nodes(blk)
    mine = {"rank": rank, "elements_same": all(_bits(el[k].cpu().numpy(), elg[k].cpu().numpy()[ge]) for k in el)}
    nbr, lists = interface_node_lists(blocks, rank)
    iface = np.zeros(F.n_nodes, dtype=bool)
    for v in lists:
        iface[v] = True
    mine["n_interface"] = int(iface.sum())
    for kind, name in ((0, "stress"), (1, "strain")):
        work, out = _raw(F, x, kind)
        workg, outg = _raw(Fg, xg, kind)
        wg, og = workg[gn], outg[gn]
        diff = np.abs(out - og)
        ulp8 = 8.0 * np.spacing(np.max(np.abs(og), axis=1))
        mine[name] = {"interior_same": _bits(out[~iface], og[~iface]), "counts_same": bool(np.array_equal(work[:, 3], wg[:, 3])),
                      "interface_within_8ulp": bool(np.all(diff[iface] <= ulp8[iface, None])),
                      "interface_max_ulps": float(np.max(diff[iface] / np.spacing(np.max(np.abs(og[iface]), axis=1))[:, None]))
                      if iface.any() else 0.0,
                      "api_same": _bits(F.nodal(x, name).cpu().numpy(), out)}
    gathered = [None] * world
    dist.gather_object(mine, gathered if rank == 0 else None, dst=0)
    if rank == 0:
        res = {"world": world, "field": field, "transport": comm.transport, "ranks": gathered}
        with open(out_path, "w") as fh:
            json.dump(res, fh)
        print(json.dumps(res))
    del F
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
