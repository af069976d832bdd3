"""Record spline outputs of the REFERENCE (pypose v0.9.5, fp64, CPU) for tests/golden/spline.npz:

    python oracle/make_golden_spline.py

TEST INFRASTRUCTURE ONLY.  Cases: `bspline` (pypose/function/spline.py:105-225) on batched SE3 poses with and without
extrapolation at two intervals; `chspline` (:5-102) on batched points at three intervals.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "spline.npz")


def main():
    torch.manual_seed(17)
    g = {}
    poses = ref.randn_SE3(3, 7, sigma=0.6, dtype=torch.float64)
    g["bspline/poses"] = poses.tensor().numpy().copy()
    for name, interval, ext in (("i02", 0.2, False), ("i03x", 0.3, True), ("i05", 0.5, False), ("i01x", 0.1, True)):
        g[f"bspline/{name}"] = ref.bspline(poses, interval, ext).tensor().numpy().copy()
    two = ref.randn_SE3(2, sigma=0.8, dtype=torch.float64)
    g["bspline/two"] = two.tensor().numpy().copy()
    g["bspline/two_i01x"] = ref.bspline(two, 0.1, True).tensor().numpy().copy()
    pts = torch.randn(2, 9, 4, dtype=torch.float64)
    g["chspline/points"] = pts.numpy().copy()
    for name, interval in (("i01", 0.1), ("i04", 0.4), ("i05", 0.5)):
        g[f"chspline/{name}"] = ref.chspline(pts, interval=interval).numpy().copy()
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, {k: v.shape for k, v in g.items()})


if __name__ == "__main__":
    main()
