"""The index-free hex-box operator across ranks (tests/hexop_dd_worker.py): 2 and 4 ranks time-sharing one GPU over the
peer transport, uniform and field boxes.  Jacobi-PCG and, on the uniform box, MG-PCG with HexMultigrid(blocks=...) give x,
resvec and trace bit-identical on every rank to the same run on the ordered EBE operator, and the Jacobi solution matches
the oracle's multi-part emulation of the reference."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("world,field", [(2, 0), (2, 1), (4, 0), (4, 1)])
def test_ranks_sharing_one_gpu(cuda, tmp_path, world, field):
    out = tmp_path / f"hexop_{world}_{field}.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29911 + 2 * world + field), os.path.join(HERE, "hexop_dd_worker.py"), str(out), "8", str(field)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                       env=dict(os.environ, PCGB_SHARED_GPU="1"))
    assert r.returncode == 0, r.stdout[-4000:]
    res = json.loads(out.read_text())
    assert res["transport"] == "peer"
    assert res["ref_flag"] == 0 and res["x_rel_err"] <= 1e-9, res
    assert len(res["ranks"]) == world
    for rk in res["ranks"]:
        assert rk["flag"] == 0 and abs(rk["iters"] - res["ref_iters"]) <= 2, rk
        assert rk["jacobi_same"] and rk["minv_same"], rk
        if not field:
            assert rk["mg_flag"] == 0 and rk["lam_same"] and rk["mg_same"], rk
