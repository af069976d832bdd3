"""World-size-2 (gloo, CPU) run of the sharded LM: pose-sharded PoseInv and residual-sharded reprojection
must reproduce the reference's single-process trajectories (tests/golden/lm.npz)."""
import os
import socket
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_sharded_lm_world2_matches_reference_and_sizes_both_exchange_forms(tmp_path, golden_lm):
    out = str(tmp_path / "dist.npz")
    port = str(_free_port())
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=port,
                   PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dist_worker.py"), out], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    logs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(logs)
    r, g = np.load(out), golden_lm
    np.testing.assert_allclose(r["poseinv_loss"], g["poseinv/trustregion/loss"], rtol=1e-5, atol=1e-20)
    np.testing.assert_allclose(r["poseinv_poses"], g["poseinv/trustregion/poses"][-1], atol=1e-9)
    for case in ("reproj", "reproj_hard"):
        np.testing.assert_allclose(r[f"{case}_loss"], g[f"{case}/trustregion/loss"], rtol=1e-6)
        np.testing.assert_allclose(r[f"{case}_poses"], g[f"{case}/trustregion/poses"][-1], atol=1e-8)
        np.testing.assert_array_equal(r[f"{case}_reject"], g[f"{case}/trustregion/reject"])
    np.testing.assert_allclose(r["pgo_loss"], g["pgo/trustregion/loss"], rtol=1e-6)
    np.testing.assert_allclose(r["pgo_poses"], g["pgo/trustregion/poses"][-1], atol=1e-7)
    np.testing.assert_allclose(r["ba_loss"], g["ba/trustregion/loss"], rtol=1e-5)
    np.testing.assert_allclose(r["ba_poses"], g["ba/trustregion/poses"][-1], atol=1e-6)
    np.testing.assert_allclose(r["ba_points"], g["ba/trustregion/points"][-1], atol=1e-6)
    assert r["regions_run"].tolist() == [9, 9]               # every rank ran as many timed regions as the slowest wanted
    # host side of the sharded reprojection exchange: rank 0 wrote the file, so `cams` is rank 0's list
    np.testing.assert_array_equal(r["present"], [[1, 0, 1, 0, 0, 1, 0], [0, 0, 1, 1, 0, 0, 0]])
    np.testing.assert_array_equal(r["cams"], [0, 2, 5])
    al = lambda n: (n + 255) // 256 * 256                    # regions are 256-byte aligned
    assert r["payload_gather"].tolist() == [0, al(2 * 1000 * 28 * 4), al(2 * 1000 * 28 * 4) + al(1000 * 8 * 4)]   # all blocks to every rank
    assert r["payload_owner"].tolist() == [0, al(2 * 500 * 28 * 4), al(2 * 500 * 28 * 4) + al(1000 * 8 * 4)]      # blocks to owners
