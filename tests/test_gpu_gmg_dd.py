"""The multigrid preconditioner across ranks (pcgb_mg_create_ranks, multigrid.HexMultigrid with `blocks`): ranks
time-sharing cuda:0 run tests/gmg_dd_worker.py, which checks the hierarchy, every part of the V-cycle, the whole V-cycle and
MG-PCG against the one-rank preconditioner of the global mesh and the host restatements; the same worker runs with one GPU
per rank on both transports."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (pgrid, elements per rank and axis, fine operator).  16 per rank on 2x2x1: rank 0's halo holds 1785 entries, more
# than one pack CTA (1024).  3x1x1: the middle rank has two neighbours and owns only one of its interfaces.
CASES = [((2, 1, 1), 8, "csr"), ((3, 1, 1), 8, "csr"), ((2, 2, 1), 8, "csr"), ((2, 2, 1), 16, "csr"),
         ((2, 1, 1), 16, "ebe_ordered"), ((2, 1, 1), 8, "ebe")]


def _run(pgrid, per, kind, tmp_path, port, env):
    world = pgrid[0] * pgrid[1] * pgrid[2]
    out = tmp_path / f"gmg_dd_{world}_{per}_{kind}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "gmg_dd_worker.py"), str(out), ",".join(map(str, pgrid)), str(per), kind]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads(out.read_text())


def _check(res, transport):
    assert res["transport"] == transport
    assert res["fails"] == [], res["fails"][:20]
    assert res["trace_complete"] and res["trace_identical"] and res["trace_replayed"] is True, res
    if transport == "peer":
        assert res["trace_sum_mismatches"] == 0 and res["trace_sum_checked"] > 0
    assert res["x_vs_ref"] <= 1e-9, res["x_vs_ref"]
    for s in res["stats"]:
        assert s["refusals"] == 4
    print(json.dumps({k: res[k] for k in ("pgrid", "per", "kind", "stats", "x_vs_ref", "seconds")}))


@pytest.mark.parametrize("pgrid,per,kind", CASES)
def test_ranks_sharing_one_gpu(cuda, tmp_path, pgrid, per, kind):
    port = 29711 + CASES.index((pgrid, per, kind))
    _check(_run(pgrid, per, kind, tmp_path, port, {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"}), "peer")


@pytest.mark.parametrize("transport", ["peer", "nccl"])
@pytest.mark.parametrize("pgrid", [(2, 1, 1), (2, 2, 1)])
def test_one_gpu_per_rank(cuda, tmp_path, pgrid, transport):
    import torch
    world = pgrid[0] * pgrid[1] * pgrid[2]
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    env = {"PCGB_COMM": "nccl"} if transport == "nccl" else {}
    _check(_run(pgrid, 8, "csr", tmp_path, 29741 + world + (10 if transport == "nccl" else 0), env), transport)
