"""Goldens for two consumers of the hot path (SURVEY.md §8f.3-4), from the REFERENCE (pypose v0.9.5, fp64 CPU):
* EPnP's Gauss-Newton refinement of beta (module/pnp.py:13-27 BetaObjective, :185-190 _refine: GaussNewton + LSTSQ +
  StopOnPlateau(steps=10, patience=3));
* the whole EPnP module (module/pnp.py:33-320) and svdtf (function/geometry.py:315-358) on random scenes;
* the g2o information-matrix layout (examples/module/pgo/pgo_dataset.py:22-29 info2mat).
    python oracle/make_golden_consumers.py     # writes tests/golden/consumers.npz
Test infrastructure only."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402
from pypose.module.pnp import BetaObjective  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "consumers.npz")


def main():
    g = torch.Generator().manual_seed(4)
    DT = torch.float64
    B = 3
    base_w = torch.randn(B, 4, 3, generator=g, dtype=DT)
    nullv = torch.linalg.qr(torch.randn(B, 12, 4, generator=g, dtype=DT))[0].mT          # (B, 4, 12) orthonormal rows
    beta_true = torch.tensor([[1.0, 0.1, -0.05, 0.02]], dtype=DT).repeat(B, 1) + 0.05 * torch.randn(B, 4, generator=g, dtype=DT)
    base_c = ref.bmv(nullv.mT, beta_true).unflatten(-1, (4, 3))
    # make the world bases consistent with the camera bases of beta_true (distances are what the objective compares)
    base_w = base_c + 0.0
    beta0 = beta_true + 0.05 * torch.randn(B, 4, generator=g, dtype=DT)
    model = BetaObjective(beta0.clone())
    optim = ref.optim.GaussNewton(model, solver=ref.optim.solver.LSTSQ())
    sched = ref.optim.scheduler.StopOnPlateau(optim, steps=10, patience=3)
    losses = []
    while sched.continual():
        loss = optim.step(input=(base_w, nullv))
        sched.step(loss)
        losses.append(float(loss))
    out = {"pnp/base_w": base_w.numpy(), "pnp/nullv": nullv.numpy(), "pnp/beta0": beta0.numpy(),
           "pnp/beta": model.beta.detach().numpy(), "pnp/loss": np.array(losses)}
    # ---- the whole EPnP module (module/pnp.py:33-320) on random scenes: exact pixels and pixels with 0.3 px of noise,
    # batch shape (2, 3), 24 points, refine on / off
    f = 600.0
    K = torch.tensor([[f, 0, 320.0], [0, 1.1 * f, 240.0], [0, 0, 1]], dtype=DT)
    pose = ref.se3(0.6 * torch.randn(2, 3, 6, generator=g, dtype=DT)).Exp()
    pc = torch.rand(2, 3, 24, 3, generator=g, dtype=DT) * torch.tensor([4.0, 3.0, 4.0], dtype=DT) + torch.tensor([-2.0, -1.5, 4.0], dtype=DT)
    pw = pose.unsqueeze(-2).Inv().Act(pc)
    pix = ref.point2pixel(pc, K)
    noisy = pix + 0.3 * torch.randn(pix.shape, generator=g, dtype=DT)
    out.update({"epnp/K": K.numpy(), "epnp/points": pw.numpy(), "epnp/pixels": pix.numpy(), "epnp/pixels_noisy": noisy.numpy(),
                "epnp/pose_true": pose.tensor().numpy()})
    for tag, px in (("exact", pix), ("noisy", noisy)):
        for refine in (False, True):
            est = ref.module.EPnP(intrinsics=K, refine=refine)(pw, px)
            out[f"epnp/{tag}/refine{int(refine)}"] = est.tensor().detach().numpy()
    src = torch.randn(4, 30, 3, generator=g, dtype=DT)
    T = ref.se3(torch.randn(4, 6, generator=g, dtype=DT)).Exp()
    out.update({"svdtf/source": src.numpy(), "svdtf/target": T.unsqueeze(-2).Act(src).numpy(),
                "svdtf/T": ref.svdtf(src, T.unsqueeze(-2).Act(src)).tensor().numpy()})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, losses)


if __name__ == "__main__":
    main()
