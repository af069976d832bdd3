"""Gradient goldens of IMUPreintegrator from the REFERENCE (pypose v0.9.5, fp64 CPU): the reference integrator is
differentiable in the signals and the initial state (its IMU-corrector training relies on it).  Inputs are the ones
already stored in tests/golden/scan_imu.npz.
    python oracle/make_golden_imu_grad.py   # writes tests/golden/imu_grad.npz
Test infrastructure only.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "..", "tests", "golden", "scan_imu.npz")
OUT = os.path.join(HERE, "..", "tests", "golden", "imu_grad.npz")


def scalar(out):
    """One scalar that touches every predicted state."""
    return (out["pos"] ** 2).sum() + (out["vel"] ** 2).sum() + (out["rot"].Log().tensor() ** 2).sum()


def main():
    g, o = np.load(SRC), {}
    t = lambda k: torch.from_numpy(g[k]).clone()
    for tag in ("free", "rot"):
        for cov in (False, True):
            dt, gyro, acc = (t(k).requires_grad_() for k in ("imu/dt", "imu/gyro", "imu/acc"))
            pos, vel = t("imu/init_pos").requires_grad_(), t("imu/init_vel").requires_grad_()
            init = {"pos": pos, "rot": ref.SO3(t("imu/init_rot")), "vel": vel}
            kw = {"rot": ref.SO3(t("imu/rot"))} if tag == "rot" else {}
            m = ref.module.IMUPreintegrator(prop_cov=cov, reset=True).double()
            out = m(dt, gyro, acc, init_state=init, **kw)
            s = scalar(out)
            s.backward()
            key = f"{tag}/{'cov' if cov else 'nocov'}"
            o[f"{key}/scalar"] = s.detach().numpy()
            for name, v in (("dt", dt), ("gyro", gyro), ("acc", acc), ("pos", pos), ("vel", vel)):
                o[f"{key}/grad_{name}"] = v.grad.numpy()
    np.savez_compressed(OUT, **o)
    print("wrote", OUT, len(o))


if __name__ == "__main__":
    main()
