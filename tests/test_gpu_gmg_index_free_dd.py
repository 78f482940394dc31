"""The index-free multigrid hierarchy across ranks (pcgb_mg_create_ranks_index_free, HexMultigrid(blocks=...,
coarse="index_free")): ranks time-sharing cuda:0 run tests/gmg_if_dd_worker.py, which checks each ranked level's local
product against the index-free operator of the rank's box, lambda against the one-rank index-free hierarchy of the global
mesh, the V-cycle against the host restatement, and MG-PCG against the one-rank iteration count and the oracle."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# 16 elements per rank and axis: ranked levels 16, 8, 4 (1 and 2 smoothed, index-free with the level's exchange-add),
# gathered at 2
CASES = [((2, 1, 1), 16, "csr"), ((2, 1, 1), 16, "hexop"), ((2, 2, 1), 16, "csr"), ((2, 2, 1), 16, "hexop")]


@pytest.mark.parametrize("pgrid,per,kind", CASES)
def test_index_free_hierarchy_on_ranks_sharing_one_gpu(cuda, tmp_path, pgrid, per, kind):
    world = pgrid[0] * pgrid[1] * pgrid[2]
    out = tmp_path / f"gmg_if_dd_{world}_{per}_{kind}.json"
    port = 29771 + CASES.index((pgrid, per, kind))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "gmg_if_dd_worker.py"), str(out), ",".join(map(str, pgrid)), str(per), kind]
    env = dict(os.environ, PCGB_SHARED_GPU="1", PCGB_EXPECT_TRANSPORT="peer")
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200, env=env)
    assert r.returncode == 0, r.stdout[-4000:]
    res = json.loads(out.read_text())
    assert res["fails"] == [], res["fails"][:20]
    assert all(s["ranked_levels_checked"] == 2 for s in res["stats"]), res["stats"]
    assert res["x_vs_ref"] <= 1e-9, res["x_vs_ref"]
    print(json.dumps({k: res[k] for k in ("pgrid", "per", "kind", "stats", "x_vs_ref", "seconds")}))
