"""Voxel models across ranks: ranks time-sharing cuda:0 run tests/voxel_dd_worker.py, where every rank builds its own field
operator from its block_field slice and Jacobi-PCG across ranks must equal the one-rank solve of the same field."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (pgrid, elements per rank and axis, contrast)
CASES = [((2, 1, 1), 8, 100.0), ((2, 2, 1), 6, 10.0)]


@pytest.mark.parametrize("pgrid,per,contrast", CASES)
def test_field_ranks_sharing_one_gpu(cuda, tmp_path, pgrid, per, contrast):
    world = pgrid[0] * pgrid[1] * pgrid[2]
    out = tmp_path / f"voxel_dd_{world}_{per}.json"
    port = 29781 + CASES.index((pgrid, per, contrast))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "voxel_dd_worker.py"), str(out), ",".join(map(str, pgrid)), str(per),
           str(contrast)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200,
                       env=dict(os.environ, PCGB_SHARED_GPU="1", PCGB_EXPECT_TRANSPORT="peer"))
    assert r.returncode == 0, r.stdout[-4000:]
    res = json.loads(out.read_text())
    assert res["fails"] == [], res["fails"][:20]
    assert len(res["stats"]) == world and all(s["refused"] for s in res["stats"])
    assert any(s["e0"][0] != 0 for s in res["stats"])       # a box off the clamped face
    assert max(s["x_vs_one_rank"] for s in res["stats"]) <= 1e-9
    print(json.dumps(res))
