"""Goldens for cumprod / IMUPreintegrator from the REFERENCE (pypose v0.9.5, fp64 CPU):
    python oracle/make_golden_scan.py   # writes tests/golden/scan_imu.npz
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "scan_imu.npz")


def main():
    torch.manual_seed(11)
    g = {}
    DT = torch.float64
    for name, rnd in (("SO3", ref.randn_SO3), ("SE3", ref.randn_SE3), ("RxSO3", ref.randn_RxSO3), ("Sim3", ref.randn_Sim3)):
        x = rnd(3, 37, sigma=0.4, dtype=DT)
        g[f"cumprod/{name}/in"] = x.numpy().copy()
        g[f"cumprod/{name}/left"] = ref.cumprod(x, dim=1, left=True).numpy()
        g[f"cumprod/{name}/right"] = ref.cumprod(x, dim=1, left=False).numpy()
    # IMU: B = 3 trajectories, F = 50 samples, with and without known rotations / covariance
    B, F = 3, 50
    dt = torch.full((B, F, 1), 0.005, dtype=DT) * (1 + 0.1 * torch.rand(B, F, 1, dtype=DT))
    gyro = 0.3 * torch.randn(B, F, 3, dtype=DT)
    acc = torch.randn(B, F, 3, dtype=DT) + torch.tensor([0, 0, 9.81], dtype=DT)
    rot = ref.randn_SO3(B, F, sigma=0.5, dtype=DT)
    init = {"pos": torch.randn(B, 1, 3, dtype=DT), "rot": ref.randn_SO3(B, 1, dtype=DT), "vel": torch.randn(B, 1, 3, dtype=DT)}
    g["imu/dt"], g["imu/gyro"], g["imu/acc"], g["imu/rot"] = dt.numpy(), gyro.numpy(), acc.numpy(), rot.numpy()
    g["imu/init_pos"], g["imu/init_rot"], g["imu/init_vel"] = init["pos"].numpy(), init["rot"].numpy(), init["vel"].numpy()
    for tag, kw in (("free", {}), ("rot", {"rot": rot})):
        m = ref.module.IMUPreintegrator(prop_cov=True, reset=True).double()
        inte = m.integrate(dt, gyro, acc, init_rot=init["rot"], **kw)
        for k, v in inte.items():
            g[f"imu/{tag}/inte/{k}"] = v.numpy() if not hasattr(v, "tensor") else v.tensor().numpy()
        out = m(dt, gyro, acc, init_state=init, **kw)
        for k, v in out.items():
            g[f"imu/{tag}/out/{k}"] = v.numpy() if not hasattr(v, "tensor") else v.tensor().numpy()
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, len(g))


if __name__ == "__main__":
    main()
