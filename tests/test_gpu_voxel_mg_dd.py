"""The voxel-model multigrid across ranks (pcgb_mg_create_ranks_field, multigrid.HexMultigrid with `blocks` and the global
E_field): ranks time-sharing cuda:0 run tests/voxel_mg_dd_worker.py, which checks the hierarchy, the V-cycle and MG-PCG
against the one-rank field hierarchy of the global mesh and the uniform ranked handle; the same worker runs with one GPU
per rank on both transports."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (pgrid, elements per rank and axis, fine operator, contrast).  Contrast 1 is a constant field, also checked against the
# uniform ranked handle.  The gathered global box (level la + 1) is itself the coarsest level on 2x1x1, 3x1x1 and 2x2x1
# (4x2x2, 6x2x2, 4x4x2 elements); on 2x2x2 (4x4x4) it is a smoothed CSR level above a 2x2x2 coarsest one.
CASES = [((2, 1, 1), 8, "csr", 1.0), ((2, 1, 1), 8, "csr", 10.0), ((2, 1, 1), 8, "csr", 100.0),
         ((3, 1, 1), 8, "csr", 100.0), ((2, 2, 1), 8, "csr", 10.0), ((2, 2, 1), 8, "csr", 100.0),
         ((2, 1, 1), 16, "csr", 100.0), ((2, 1, 1), 16, "ebe_ordered", 10.0), ((2, 2, 1), 8, "box", 100.0),
         ((3, 1, 1), 8, "box", 1.0), ((2, 2, 2), 8, "csr", 100.0)]


def _run(pgrid, per, kind, contrast, tmp_path, port, env):
    world = pgrid[0] * pgrid[1] * pgrid[2]
    out = tmp_path / f"voxel_mg_dd_{world}_{per}_{kind}_{contrast:g}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "voxel_mg_dd_worker.py"), str(out), ",".join(map(str, pgrid)), str(per),
           kind, str(contrast)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads(out.read_text())


def _check(res, transport):
    assert res["transport"] == transport
    assert res["fails"] == [], res["fails"][:20]
    for s in res["stats"]:
        assert s["refusals"] == 5
        assert s["iters"] == s["iters_one_rank"] and 2 * s["iters"] < s["iters_jacobi"], s
    print(json.dumps({k: res[k] for k in ("pgrid", "per", "kind", "contrast", "stats", "seconds")}))


@pytest.mark.parametrize("pgrid,per,kind,contrast", CASES)
def test_ranks_sharing_one_gpu(cuda, tmp_path, pgrid, per, kind, contrast):
    port = 29611 + CASES.index((pgrid, per, kind, contrast))
    _check(_run(pgrid, per, kind, contrast, tmp_path, port, {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"}), "peer")


@pytest.mark.parametrize("transport", ["peer", "nccl"])
@pytest.mark.parametrize("pgrid", [(2, 1, 1), (2, 2, 1)])
def test_one_gpu_per_rank(cuda, tmp_path, pgrid, transport):
    import torch
    world = pgrid[0] * pgrid[1] * pgrid[2]
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    env = {"PCGB_COMM": "nccl"} if transport == "nccl" else {}
    _check(_run(pgrid, 8, "csr", 100.0, tmp_path, 29641 + world + (10 if transport == "nccl" else 0), env), transport)
