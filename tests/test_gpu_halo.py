"""The exchange between ranks kernel by kernel: the peer halo pack / unpack (k_halo_pack_peer, k_halo_unpack_peer), the peer
all-reduce (k_allreduce_peer, cta_allreduce) and the NCCL halo (k_halo_pack, k_halo_unpack_add), bit for bit against the
host reference of tests/halo_cases.py on synthetic plans that cross the pack and unpack CTA edges (tests/halo_worker.py);
and pcgb_halo_create's refusals, which must come before anything is allocated."""
import gc
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import halo_cases as H

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(world, tmp_path, port, env):
    out = tmp_path / f"halo_{world}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "halo_worker.py"), str(out), "all"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads(out.read_text())


def _check(res, world, transport):
    assert res["transport"] == transport
    assert res["cases"] == H.cases_of(world)
    assert res["fails"] == [], res["fails"][:20]
    ncase = len(H.cases_of(world))
    for c in res["counts"]:
        assert c["exchange"] == 6 * ncase and c["apply"] == ncase and c["jacobi"] >= 1
        assert c["alternate"] == 6 and c["allreduce"] >= 9 + 6
        if transport == "peer":
            assert c["refusal"] == 3          # count 9, the asymmetric table, the count mismatch


@pytest.mark.parametrize("world", [2, 3, 4])
def test_exchange_bitwise_ranks_sharing_one_gpu(cuda, tmp_path, world):
    """`world` OS processes time-share cuda:0 over a peer-only communicator: every case of that world, with its
    exchanges, applications, Jacobi, alternating plans, all-reduces and refusals, bit for bit on every rank."""
    res = _run(world, tmp_path, 29917 + world, {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"})
    _check(res, world, "peer")


@pytest.mark.parametrize("world", [2, 3, 4])
def test_exchange_bitwise_nccl(cuda, tmp_path, world):
    """The same worker on the NCCL transport, one GPU per rank (k_halo_pack, ncclSend/Recv, k_halo_unpack_add)."""
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    res = _run(world, tmp_path, 29937 + world, {"PCGB_COMM": "nccl", "PCGB_EXPECT_TRANSPORT": "nccl"})
    _check(res, world, "nccl")


def test_create_refusals_allocate_nothing(cuda):
    """pcgb_halo_create refuses a duplicate neighbour, a duplicate index in one list, a neighbour equal to this rank, below 0
    or at nranks, and an index out of range (the host restatement halo_cases.refusal agrees), before it allocates; an empty
    list is dropped, so rank 0 of a plan whose lists are all empty has no neighbours."""
    import torch
    from pcg_mpi_solver_b200 import _lib
    from pcg_mpi_solver_b200.csr import CsrMatrix
    from pcg_mpi_solver_b200.solver import Communicator, SubdomainOperator
    comm = Communicator(0, 4, None)              # no window exchange: nothing collective runs
    bad = H.refused_plans()
    n = next(iter(bad.values()))[2]
    r = torch.arange(n + 1, dtype=torch.int32, device=cuda)
    A = CsrMatrix(r, r[:n].clone(), torch.ones(n, dtype=torch.float64, device=cuda), (n, n))
    ok = SubdomainOperator(A, comm, [3, 1], [np.zeros(0, np.int64), np.arange(5)])   # warm-up; the empty list is dropped
    assert ok.halo_bytes() == 8 * 5
    del ok
    gc.collect()
    msgs = {"duplicate_neighbour": "listed twice", "duplicate_index": "appears twice", "neighbour_self": "bad neighbour table",
            "neighbour_negative": "bad neighbour table", "neighbour_nranks": "bad neighbour table",
            "index_out_of_range": "out of range", "index_negative": "out of range"}
    for name, (nbr, lists, n_) in bad.items():
        assert H.refusal({"world": 4, "n": [n_], "nbr": [nbr], "lists": [lists]}, 0) == msgs[name]
        for _ in range(3):
            torch.cuda.synchronize()
            free0, _ = torch.cuda.mem_get_info(cuda)
            with pytest.raises(_lib.PcgbError, match=r"\(-1\).*" + msgs[name]):
                SubdomainOperator(A, comm, nbr, lists)
            gc.collect()
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info(cuda)[0] >= free0, name
