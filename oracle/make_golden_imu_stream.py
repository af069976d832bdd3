"""Streaming goldens of IMUPreintegrator from the REFERENCE (pypose v0.9.5, fp64 CPU): the default constructor
(reset=False, prop_cov=True) carries pos / rot / vel / cov / Rij from one call to the next, which is how the reference's
examples feed consecutive IMU windows.  B = 3 trajectories, three windows of 50, 1 and 77 samples; the second window
passes its own gyro_cov / acc_cov.  The run is repeated with known rotations (`rot`).
    PYPOSE_REFERENCE=<pypose checkout> python oracle/make_golden_imu_stream.py   # writes tests/golden/imu_stream.npz
Test infrastructure only.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "imu_stream.npz")
B, WINDOWS = 3, (50, 1, 77)


def main():
    torch.manual_seed(23)
    DT = torch.float64
    g = {}
    for w, F in enumerate(WINDOWS):
        g[f"in/{w}/dt"] = (0.005 * (1 + 0.1 * torch.rand(B, F, 1, dtype=DT))).numpy()
        g[f"in/{w}/gyro"] = (0.3 * torch.randn(B, F, 3, dtype=DT)).numpy()
        g[f"in/{w}/acc"] = (torch.randn(B, F, 3, dtype=DT) + torch.tensor([0, 0, 9.81], dtype=DT)).numpy()
        g[f"in/{w}/rot"] = ref.randn_SO3(B, F, sigma=0.5, dtype=DT).numpy()
    g["in/1/gyro_cov"] = (1e-5 * (1 + torch.rand(B, 1, 3, dtype=DT))).numpy()
    g["in/1/acc_cov"] = (4e-3 * (1 + torch.rand(B, 1, 3, dtype=DT))).numpy()
    for tag in ("free", "rot"):
        m = ref.module.IMUPreintegrator().double()
        for w in range(len(WINDOWS)):
            t = lambda k: torch.from_numpy(g[f"in/{w}/{k}"])
            kw = {"rot": ref.SO3(t("rot"))} if tag == "rot" else {}
            if w == 1:
                kw.update(gyro_cov=t("gyro_cov"), acc_cov=t("acc_cov"))
            out = m(t("dt"), t("gyro"), t("acc"), **kw)
            for k in ("pos", "vel", "rot", "cov"):
                v = out[k]
                g[f"{tag}/{w}/out/{k}"] = (v.tensor() if hasattr(v, "tensor") else v).numpy().copy()
            for k in ("pos", "rot", "vel", "cov", "Rij"):
                v = getattr(m, k)
                g[f"{tag}/{w}/state/{k}"] = (v.tensor() if hasattr(v, "tensor") else v).numpy().copy()
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, len(g))


if __name__ == "__main__":
    main()
