"""The rap voxel multigrid across ranks (pcgb_mg_create_ranks_field_rap, HexMultigrid(coarse="rap") with `blocks` and the
global E_field): ranks time-sharing cuda:0 run tests/voxel_rap_dd_worker.py, which checks the hierarchy, the V-cycle and
MG-PCG against the ranked field hierarchy on the same split and the one-rank rap handle of the global mesh; the same
worker runs with one GPU per rank on both transports."""
import json
import math
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (split, combos of fine operator and contrast).  2x1x1 of 8^3: la = 2, level 2 is the gathered level.  16^3 per rank: la = 3,
# a ranked CSR level 2; the middle rank of 3x1x1 has a level-1 box with a free low-x face and neighbours on both x sides.
# The x tiling 24 + 8 of 32x16x16 has level-1 widths 12 and 4, neither free-node count a multiple of the 8-node brick.
CASES = [("grid:2,1,1:8", "csr:1,box:10,csr:100"),
         ("grid:2,1,1:16", "box:1,csr:10,box:100"),
         ("grid:3,1,1:16", "csr:1,box:10,csr:100"),
         ("grid:2,2,1:16", "box:10,csr:100"),
         ("grid:2,2,2:16", "csr:10,box:100"),
         ("tile:32,16,16:24,8", "csr:1,box:10,csr:100,box:100")]


def _world(split):
    if split == "large":
        return 2
    kind, a, b = split.split(":")
    return math.prod(int(v) for v in a.split(",")) if kind == "grid" else len(b.split(","))


def _run(split, combos, tmp_path, port, env):
    world = _world(split)
    out = tmp_path / "voxel_rap_dd.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "voxel_rap_dd_worker.py"), str(out), split] + ([combos] if combos else [])
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-4000:]
    return json.loads(out.read_text())


def _check(res, transport, ncombos):
    assert res["transport"] == transport
    assert res["fails"] == [], res["fails"][:20]
    for per_rank in res["stats"]:
        assert len(per_rank) == ncombos
        for s in per_rank:
            if "skipped" not in s:
                assert s["iters"] == s["iters_one_rank"], s
    print(json.dumps({k: res[k] for k in ("split", "stats", "seconds")}))


@pytest.mark.parametrize("split,combos", CASES)
def test_ranks_sharing_one_gpu(cuda, tmp_path, split, combos):
    res = _run(split, combos, tmp_path, 29711 + [c[0] for c in CASES].index(split),
               {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"})
    _check(res, "peer", len(combos.split(",")))
    assert all(s[-1]["refusals"] == 3 for s in res["stats"])


def test_two_ranks_of_256_cubed_against_one_rank(cuda, tmp_path):
    """512x256x256 as 2x1x1 ranks of 256^3 against the one-rank rap handle of the whole mesh (skipped below 60 GB free):
    equal iterations, x within 1e-9, the free-memory drop within 2 % of rap_rank_bytes plus the fields."""
    _check(_run("large", None, tmp_path, 29731, {"PCGB_SHARED_GPU": "1", "PCGB_EXPECT_TRANSPORT": "peer"}), "peer", 1)


@pytest.mark.parametrize("transport", ["peer", "nccl"])
@pytest.mark.parametrize("split", ["grid:2,1,1:16", "grid:2,2,1:16"])
def test_one_gpu_per_rank(cuda, tmp_path, split, transport):
    import torch
    world = _world(split)
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    env = {"PCGB_COMM": "nccl"} if transport == "nccl" else {}
    _check(_run(split, "csr:100", tmp_path, 29741 + world + (10 if transport == "nccl" else 0), env), transport, 1)
