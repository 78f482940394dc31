"""Multi-rank worker for the halo exchange-add and the all-reduce (launched by tests/test_gpu_halo.py through
torch.distributed.run).

Every rank builds each synthetic plan of its world (tests/halo_cases.py) as a SubdomainOperator over an identity
CsrMatrix, so only the halo acts, and checks bit for bit against the host reference on every rank:
- exchange_add six times in a row with fresh y (odd and even epochs; a read of the wrong parity half sees the data of the
  exchange before last), apply(x) = x + exchange, and jacobi() = 1 / (1 + multiplicity);
- two plans alternating on one communicator, with all-reduces between their exchanges;
- Communicator.allreduce_sum: counts 0 to 8 (peer transport: the rank-order sum from 0.0, bit for bit), cancelling values,
  inf and NaN, and on a peer-only communicator a refused count of 9 followed by a correct all-reduce;
- import refusals (peer transport): asymmetric tables and count mismatches raise PcgbError on every rank.
Ranks never raise on a mismatch: they record it, so all ranks stay in step, and rank 0 writes every rank's findings."""
import datetime
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist

from tests import halo_cases as H


def _ys(p, seed):
    """Fresh values for every rank (every rank draws all of them, so each can compute its own expected result)."""
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(n) * 2.0 ** rng.integers(-30, 31, n) for n in p["n"]]


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def main():
    out_path = sys.argv[1]
    only = sys.argv[2].split(",") if len(sys.argv) > 2 and sys.argv[2] != "all" else None
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = os.environ.get("PCGB_SHARED_GPU", "0") == "1"     # all ranks on cuda:0, peer-only communicator
    if shared:
        local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    timeout = datetime.timedelta(seconds=120)                  # a host-side mismatch fails in minutes, not half an hour
    if shared:
        dist.init_process_group("gloo", timeout=timeout)
    else:
        dist.init_process_group("nccl", device_id=dev, timeout=timeout)
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator.from_torch_distributed(dev, nccl=not shared)
    transport = comm.transport
    if os.environ.get("PCGB_EXPECT_TRANSPORT"):
        assert transport == os.environ["PCGB_EXPECT_TRANSPORT"], (transport, comm.peer_error)
    peer = transport == "peer"
    fails, counts = [], {"exchange": 0, "apply": 0, "jacobi": 0, "alternate": 0, "allreduce": 0, "refusal": 0}
    t0 = time.time()

    def check(what, got, want):
        if not _same(got, want):
            g, w = np.asarray(got), np.asarray(want)
            bad = int(np.sum(g != w)) if g.shape == w.shape else -1
            fails.append(f"rank {rank} {what}: {bad} entries differ")

    def identity(n):
        r = torch.arange(n + 1, dtype=torch.int32, device=dev)
        return CsrMatrix(r, r[:n].clone(), torch.ones(n, dtype=torch.float64, device=dev), (n, n))

    def build(p):
        return SubdomainOperator(identity(p["n"][rank]), comm, p["nbr"][rank], p["lists"][rank])

    def t(v):
        return torch.from_numpy(np.ascontiguousarray(v)).to(dev)

    names = [k for k in H.cases_of(world) if only is None or k in only]
    ops, plans = {}, {}
    for ci, name in enumerate(names):
        p = H.plan(name)
        op = build(p)
        ops[name], plans[name] = op, p
        if op.halo_bytes() != 8 * H.m_of(p, rank):
            fails.append(f"rank {rank} {name}: halo_bytes {op.halo_bytes()} != 8 * {H.m_of(p, rank)}")
        for call in range(6):
            ys = _ys(p, 1000 * ci + call)
            y = t(ys[rank])
            op.exchange_add(y)
            check(f"{name} exchange {call}", y.cpu().numpy(), H.expected(ys, p, [rank])[0])
            counts["exchange"] += 1
        xs = _ys(p, 1000 * ci + 99)
        check(f"{name} apply", op.apply(t(xs[rank])).cpu().numpy(), H.expected(xs, p, [rank])[0])
        counts["apply"] += 1
        if name in ("w3_empty", "w4_hub", "w2_1025"):
            ones = [np.ones(n) for n in p["n"]]
            check(f"{name} jacobi", op.jacobi().cpu().numpy(), 1.0 / H.expected(ones, p, [rank])[0])
            counts["jacobi"] += 1
    torch.cuda.synchronize()

    def allreduce(vals, count, what):
        """vals: [world][8] values; all-reduce the first `count` of them, the rest of the buffer must stay untouched."""
        buf = t(np.concatenate([vals[rank][:count], np.full(8 - count, 7.25)]))
        with torch.cuda.device(dev):             # the library call itself: an empty tensor has no address to pass
            _lib.check(_lib.load().pcgb_allreduce_sum(comm.handle, buf.data_ptr(), count, _lib.stream_ptr()), "pcgb_allreduce_sum")
        got = buf.cpu().numpy()
        want = np.zeros(count)
        for k in range(count):
            s = 0.0
            for r in range(world):              # rank order from 0.0: the peer all-reduce's documented order
                s += float(vals[r][k])
            want[k] = s
        if peer:
            check(what, got[:count], want)
        else:                                     # NCCL adds in its own order
            mag = np.sum(np.abs([v[:count] for v in vals]), axis=0) if count else np.zeros(0)
            if not np.all(np.abs(got[:count] - want) <= world * 2.0 ** -52 * mag):
                fails.append(f"rank {rank} {what}: NCCL sum off by more than rounding")
        check(what + " tail", got[count:], np.full(8 - count, 7.25))
        counts["allreduce"] += 1

    rng = np.random.default_rng(7)
    for count in range(9):
        allreduce(rng.standard_normal((world, 8)) * 2.0 ** rng.integers(-20, 21, (world, 8)), count, f"allreduce count {count}")
    if peer:
        big = 2.0 ** 53
        pattern = [big, 1.0, -big, 1.0, -1.0, 3.0, -big, big]
        allreduce([[pattern[(r + k) % 8] for k in range(8)] for r in range(world)], 8, "allreduce cancelling")
        inf = float("inf")
        special = np.ones((world, 8))
        special[0, 0] = inf                                         # inf
        special[0, 1], special[world - 1, 1] = inf, -inf            # inf - inf = NaN
        special[1, 2] = -inf                                        # -inf
        special[world - 1, 3] = float("nan")                        # NaN from the last rank
        allreduce(special, 8, "allreduce inf/nan")
    if peer and not comm._has_nccl:
        buf = t(np.arange(9.0))
        try:
            comm.allreduce_sum(buf)
            fails.append(f"rank {rank}: count 9 accepted on a peer-only communicator")
        except _lib.PcgbError as e:
            if "(-3)" not in str(e):
                fails.append(f"rank {rank}: count 9 refused with {e}")
        check("count 9 leaves the buffer", buf.cpu().numpy(), np.arange(9.0))
        allreduce(rng.standard_normal((world, 8)), 5, "allreduce after the refused count")
        counts["refusal"] += 1

    # two plans on one communicator, alternating, with all-reduces between their exchanges (they share the window epoch)
    pair = names[:2]
    if len(pair) == 2:
        for call in range(6):
            name = pair[call % 2]
            p, op = plans[name], ops[name]
            ys = _ys(p, 5000 + call)
            y = t(ys[rank])
            op.exchange_add(y)
            check(f"alternate {name} {call}", y.cpu().numpy(), H.expected(ys, p, [rank])[0])
            allreduce(rng.standard_normal((world, 8)), 1 + call, f"allreduce between exchanges {call}")
            counts["alternate"] += 1
    ops.clear()

    # import refusals: host side only, no kernel runs; every rank must raise (a communicator with NCCL would fall back to it)
    if peer and not comm._has_nccl and only is None:
        for what, c01, c10 in (("asymmetric", 3, None), ("count mismatch", 3, 4)):
            n = 16
            nbr, lists = [], []
            if rank == 0:
                nbr, lists = [1], [np.arange(c01)]
            elif rank == 1 and c10 is not None:
                nbr, lists = [0], [np.arange(c10)]
            try:
                SubdomainOperator(identity(n), comm, nbr, lists)
                fails.append(f"rank {rank} {what}: import accepted")
            except _lib.PcgbError:
                counts["refusal"] += 1
    torch.cuda.synchronize()
    status = _lib.load().pcgb_comm_status(comm.handle, _lib.stream_ptr())
    if status != 0:
        fails.append(f"rank {rank}: communicator status {status}")
    gathered = [None] * world
    dist.gather_object({"fails": fails, "counts": counts, "seconds": time.time() - t0}, gathered if rank == 0 else None, dst=0)
    if rank == 0:
        res = {"world": world, "transport": transport, "cases": names, "fails": [f for g in gathered for f in g["fails"]],
               "counts": [g["counts"] for g in gathered], "seconds": max(g["seconds"] for g in gathered)}
        with open(out_path, "w") as f:
            json.dump(res, f)
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
