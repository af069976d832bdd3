"""Golden for the reference's `LocalBundleAdjustment` example (examples/module/reprojpgo/reprojpgo.py:16-28, 60-80): ONE
relative pose + N depths as parameters, residual reprojerr(pixel2point(pts1, depth, K), pts2, K, T.Inv()), optimised with
LM(Cholesky, TrustRegion(radius=1e3), Huber(0.1) + FastTriggs, min=1e-8, reject=128) under StopOnPlateau(steps=25,
patience=4, decreasing=1e-6) — run with the REFERENCE (pypose v0.9.5, fp64 CPU) on a synthetic frame pair.
    python oracle/make_golden_localba.py     # writes tests/golden/localba.npz
Test infrastructure only."""
import os
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as pp  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "localba.npz")


class LocalBundleAdjustment(nn.Module):          # the example's module, verbatim interface
    def __init__(self, K, pts1, pts2, depth, init_T):
        super().__init__()
        self.register_buffer("K", K)
        self.register_buffer("pts1", pts1)
        self.register_buffer("pts2", pts2)
        self.T = pp.Parameter(init_T)
        self.depth = nn.Parameter(depth)

    def forward(self):
        pts3d = pp.pixel2point(self.pts1, self.depth, self.K)
        return pp.reprojerr(pts3d, self.pts2, self.K, self.T.Inv(), reduction='none')


def main():
    g = torch.Generator().manual_seed(12)
    DT = torch.float64
    N = 60
    K = torch.tensor([[320., 0., 320.], [0., 320., 240.], [0., 0., 1.]], dtype=DT)
    depth = 2.0 + 4.0 * torch.rand(N, generator=g, dtype=DT)
    pts1 = torch.rand(N, 2, generator=g, dtype=DT) * torch.tensor([600.0, 440.0], dtype=DT) + 20.0
    motion = pp.se3(torch.tensor([0.2, -0.1, 0.15, 0.03, -0.05, 0.02], dtype=DT)).Exp()       # frame 1 -> frame 2 camera motion
    pts3d = pp.pixel2point(pts1, depth, K)
    pts2 = pp.point2pixel(pts3d, K, motion.Inv()) + 0.2 * torch.randn(N, 2, generator=g, dtype=DT)
    pts2[::11] += 6.0                                                                           # a few outlier matches
    init_T = motion * pp.se3(0.1 * torch.randn(6, generator=g, dtype=DT)).Exp()
    depth0 = depth + 0.1 * torch.randn(N, generator=g, dtype=DT)
    graph = LocalBundleAdjustment(K, pts1, pts2, depth0.clone(), init_T.clone())
    kernel = pp.optim.kernel.Huber(delta=0.1)
    opt = pp.optim.LM(graph, solver=pp.optim.solver.Cholesky(), strategy=pp.optim.strategy.TrustRegion(radius=1e3), kernel=kernel,
                      corrector=pp.optim.corrector.FastTriggs(kernel), min=1e-8, reject=128, vectorize=True)
    sched = pp.optim.scheduler.StopOnPlateau(opt, steps=25, patience=4, decreasing=1e-6)
    losses, Ts = [], []
    while sched.continual():
        loss = opt.step(input=())
        sched.step(loss)
        losses.append(float(loss))
        Ts.append(graph.T.detach().tensor().numpy().copy())
    np.savez_compressed(OUT, K=K.numpy(), pts1=pts1.numpy(), pts2=pts2.numpy(), depth0=depth0.numpy(), T0=init_T.tensor().numpy(),
                        motion=motion.tensor().numpy(), loss=np.array(losses), T=np.stack(Ts), depth=graph.depth.detach().numpy())
    print("wrote", OUT, len(losses), losses[:3], losses[-1])


if __name__ == "__main__":
    main()
