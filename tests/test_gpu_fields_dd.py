"""Field recovery across ranks (tests/fields_dd_worker.py): 2 and 4 ranks time-sharing one GPU over the peer transport,
uniform and with a global field sliced per box.  Every rank's element fields are its slice of the one-rank run on the
whole mesh bit for bit; its nodal averages too at the nodes no other rank holds, and at interface nodes the counts are
exact and the values within 8 ulp (the partial sums of three or more ranks meet in another order)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("world,field", [(2, 0), (2, 1), (4, 0), (4, 1)])
def test_ranks_sharing_one_gpu(cuda, tmp_path, world, field):
    out = tmp_path / f"fields_{world}_{field}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29951 + 2 * world + field), os.path.join(HERE, "fields_dd_worker.py"), str(out), str(field)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                       env=dict(os.environ, PCGB_SHARED_GPU="1"))
    assert r.returncode == 0, r.stdout[-4000:]
    res = json.loads(out.read_text())
    assert res["transport"] == "peer"
    assert len(res["ranks"]) == world
    for rk in res["ranks"]:
        assert rk["elements_same"] and rk["n_interface"] > 0, rk
        for kind in ("stress", "strain"):
            k = rk[kind]
            assert k["interior_same"] and k["counts_same"] and k["interface_within_8ulp"] and k["api_same"], rk
