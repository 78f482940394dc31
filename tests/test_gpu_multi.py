"""Multi-GPU parity (NCCL halo exchange-add + allreduce) against the oracle's multi-part emulation of the
reference.  Needs >= 2 GPUs on the box; skipped otherwise (the driver's 1-GPU run skips it)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(world, tmp_path, block=6, graph=1, port=29517, env=None, timeout=600, operator="csr", tol=1e-12):
    out = tmp_path / f"mgpu_{world}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "mgpu_worker.py"), str(out), str(block), str(graph), operator, repr(tol)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads(out.read_text())


def _check(res):
    summary = {k: res[k] for k in ("tol", "flag", "ref_flag", "iters", "ref_iters", "relres", "ref_relres", "y_rel_err", "x_rel_err")}
    assert res["flag"] == res["ref_flag"] == 0, summary
    assert abs(res["iters"] - res["ref_iters"]) <= 2, summary
    assert res["relres"] <= res["tol"]
    assert res["y_rel_err"] <= 1e-13          # operator + interface sum
    assert res["x_rel_err"] <= 1e3 * res["tol"]   # solution: 1e-9 at tol 1e-12
    assert res["copy_mismatch"] <= 1e-12      # shared dofs stay consistent across ranks
    assert res["weight_sum"] == res["n_global"]  # ownership weights partition the free dofs
    assert all(tuple(i) == tuple(res["all_infos"][0]) for i in res["all_infos"])  # every rank agrees
    # the loop trace: complete, bit-identical on every rank, replayed by the host restatement of the control logic, and on the
    # peer transport every reduced value is the rank-order sum of the ranks' local values
    assert res["trace_records"] > 0 and res["trace_complete"] and res["trace_identical"]
    assert res["trace_replayed"] is True, res["trace_replayed"]
    if res["transport"] == "peer":
        assert res["trace_sum_checked"] > 0 and res["trace_sum_mismatches"] == 0, (res["trace_sum_checked"], res["trace_sum_mismatches"])


# (world, graph, block, operator, PCGB_FORK, PCGB_OVERLAP); None keeps the library default (fork on, overlap off).
# Blocks 20 (2 ranks, m = ndof = 1386 on rank 0) and 16 (4 ranks) put more than one CTA into the halo pack (1024 entries
# each) and unpack (256 dofs each); the tiny blocks never leave the first.
SHARED = [(2, 1, 6, "csr", None, None), (2, 0, 6, "csr", None, None), (4, 1, 5, "csr", None, None),
          (2, 1, 6, "ebe", None, None), (2, 0, 6, "ebe", None, None), (4, 1, 5, "ebe", None, None)]
SHARED += [(w, 1, b, "csr", fork, overlap) for w, b in ((2, 20), (4, 16)) for overlap in (0, 1) for fork in (0, 1)]
SHARED += [(4, 1, 16, "ebe_ordered", None, None)]
_SHARED_RUNS = {}


def _shared_id(w, g, b, op, fork, overlap):
    base = f"{w}-{g}-{b}" if op == "csr" else f"{op}-{w}-{g}-{b}"
    return base if fork is None else f"{base}-fork{fork}-overlap{overlap}"


def _run_shared(world, tmp_path, graph, block, operator, fork, overlap):
    key = (world, graph, block, operator, fork, overlap)
    if key not in _SHARED_RUNS:
        env = {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"}
        if fork is not None:
            env.update(PCGB_FORK=str(fork), PCGB_OVERLAP=str(overlap))
        port = 29617 + 2 * world + graph + {"csr": 0, "ebe": 100, "ebe_ordered": 140}[operator] + (0 if fork is None else 200 + 10 * world + 4 * overlap + 2 * fork)
        d = tmp_path / ("fork%s-overlap%s" % (fork, overlap))
        d.mkdir(exist_ok=True)
        tol = 1e-12 if block < 16 else 1e-10
        _SHARED_RUNS[key] = _run(world, d, block=block, graph=graph, port=port, env=env, timeout=900, operator=operator, tol=tol)
    return _SHARED_RUNS[key]


@pytest.mark.parametrize("world,graph,block,operator,fork,overlap", SHARED, ids=[_shared_id(*s) for s in SHARED])
def test_peer_transport_ranks_sharing_one_gpu(cuda, tmp_path, world, graph, block, operator, fork, overlap):
    """a13/a14 on a ONE-GPU box: `world` OS processes time-share cuda:0 and exchange through CUDA-IPC mapped memory with the
    same kernels that run over NVLink between GPUs (fused all-reduce in k_reduce_ar, k_halo_pack_peer / k_halo_unpack_peer,
    interface-first SpMV split), against the oracle's multi-part emulation of the reference (pcg_solver.py:303-334, 622-628).
    operator "ebe": the matrix-free operator with its separate, unweighted p.q dot of the local product; "ebe_ordered": the
    bit-reproducible one.  With PCGB_FORK set: the halo pack and unpack run at least two CTAs, PCGB_OVERLAP=1 really splits
    the product interface-first, and the fork (the unpack on a second stream) changes no bit of x or of the trace."""
    res = _run_shared(world, tmp_path, graph, block, operator, fork, overlap)
    assert res["transport"] == "peer"
    _check(res)
    if block >= 16:
        assert min(-(-m // 1024) for m in res["halo_m"]) >= 2, res["halo_m"]            # pack CTAs of every rank
        assert min(-(-n // 256) for n in res["halo_ndof"]) >= 2, res["halo_ndof"]        # unpack CTAs of every rank
    if fork is None:
        return
    if overlap:
        assert res["plan"]["interface_tiles"] > 0, res["plan"]
    # the fork only moves the unpack to another stream: both settings give the same bits on every rank
    other = _run_shared(world, tmp_path, graph, block, operator, 1 - fork, overlap)
    assert other["x_sha"] == res["x_sha"] and other["trace_sha"] == res["trace_sha"]


MULTI = [(w, g, op) for op in ("csr", "ebe") for w, g in [(2, 1), (2, 0), (4, 1), (8, 1)]]


@pytest.mark.parametrize("transport", ["peer", "nccl"])
@pytest.mark.parametrize("world,graph,operator", MULTI, ids=[f"{w}-{g}" if op == "csr" else f"{op}-{w}-{g}" for w, g, op in MULTI])
def test_multi_gpu_matches_oracle(cuda, tmp_path, world, graph, operator, transport):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    res = _run(world, tmp_path, graph=graph, port=29517 + world + graph + (40 if transport == "nccl" else 0) + (300 if operator == "ebe" else 0),
               env={"PCGB_COMM": transport, "PCGB_EXPECT_TRANSPORT": transport}, operator=operator)
    assert res["transport"] == transport
    _check(res)


def test_concrete_8gpu_matches_reference_8rank_run(cuda, tmp_path):
    """Config C4: concrete.zip, 8-way METIS, one part per GPU, vs the reference's own 8-rank run (golden G6)."""
    import torch
    if torch.cuda.device_count() < 8:
        pytest.skip("needs 8 GPUs")
    root = os.path.dirname(HERE)
    zp = os.path.join(root, "oracle", "_ref", "concrete.zip")
    if not os.path.exists(zp):
        pytest.skip("data/concrete.zip not staged")
    out = tmp_path / "concrete8.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=8", "--master-addr", "127.0.0.1",
           "--master-port", "29571", os.path.join(HERE, "mgpu_worker.py"), str(out), "concrete", zp]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    res = json.loads(out.read_text())
    ref = res["ref"]
    assert res["flag"] == ref["Flag"] == 0 and abs(res["iters"] - ref["Iter"]) <= 2 and res["relres"] <= 1e-7
    assert abs(res["norm_u"] - ref["norm2_U"]) <= 1e-7 * ref["norm2_U"]
    assert res["sample_err"] <= 1e-6
