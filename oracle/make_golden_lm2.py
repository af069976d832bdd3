"""Trajectories of the REFERENCE's dense LM (pypose v0.9.5, fp64, CPU) on the two-pose reprojection model
(BASELINE.json configs[4] as stated; SURVEY.md §8d cfg 5-full):

    r_k = proj(T_b^-1 T_a p_k) - z_k

with (i) README.md:170-178 `project` (proj(y) = -y[:2]/y[2]) and (ii) intrinsics K through the reference's
`pp.point2pixel` (function/geometry.py:60-112).  N = 24 poses on a smooth trajectory, banded covisibility b = a + U{1..3},
~15 residual rows per pair, TrustRegion and Constant strategies.
    python oracle/make_golden_lm2.py        # writes tests/golden/lm2.npz
Test infrastructure only.
"""
import os
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "lm2.npz")


class TwoPoseReproj(nn.Module):
    def __init__(self, poses, K=None):
        super().__init__()
        self.poses = ref.Parameter(poses)
        self.K = K

    def forward(self, points, pixels, ia, ib):
        y = (self.poses[ib].Inv() @ self.poses[ia]).Act(points)
        if self.K is None:
            return -y[..., :2] / y[..., 2:] - pixels
        return ref.point2pixel(y, self.K) - pixels


def problem(seed, N=24, per_pair=15):
    g = torch.Generator().manual_seed(seed)
    DT = torch.float64
    step = ref.se3(torch.tensor([[0.3, 0.02, 0.0, 0.0, 0.05, 0.02]], dtype=DT).repeat(N, 1)
                   + 0.02 * torch.randn(N, 6, generator=g, dtype=DT)).Exp()
    gt = ref.cumprod(step, dim=0, left=False)
    ia, ib = [], []
    for a in range(N):
        for d in (1, 2, 3):
            if a + d < N and (d == 1 or torch.rand(1, generator=g).item() < 0.6):
                ia += [a] * per_pair
                ib += [a + d] * per_pair
    ia, ib = torch.tensor(ia), torch.tensor(ib)
    m = len(ia)
    # points in front of camera b, expressed in the frame of pose a
    yb = torch.rand(m, 3, generator=g, dtype=DT) * torch.tensor([4.0, 4.0, 4.0], dtype=DT) + torch.tensor([-2.0, -2.0, 2.0], dtype=DT)
    pts = (gt[ia].Inv() @ gt[ib]).Act(yb)
    perm = torch.randperm(m, generator=g)           # rows arrive unsorted
    return gt, pts[perm], yb[perm], ia[perm], ib[perm], g


def run(model, inp, strategy, steps):
    opt = ref.optim.LM(model, strategy=strategy)
    loss, poses, rej = [], [], []
    for _ in range(steps):
        loss.append(float(opt.step(inp)))
        poses.append(model.poses.detach().clone().numpy())
        rej.append(opt.reject_count)
    return np.array(loss), np.stack(poses), np.array(rej)


def main():
    out = {}
    DT = torch.float64
    gt, pts, yb, ia, ib, g = problem(7)
    N = gt.shape[0]
    init = ref.se3(0.03 * torch.randn(N, 6, generator=g, dtype=DT)).Exp() * gt
    K = torch.tensor([[320.0, 0.5, 310.0], [0.0, 300.0, 250.0], [0.0, 0.0, 1.0]], dtype=DT)
    out["gt"], out["poses0"], out["pts"], out["ia"], out["ib"], out["K"] = gt.numpy(), init.numpy(), pts.numpy(), ia.numpy(), ib.numpy(), K.numpy()
    noise = 1e-3 * torch.randn(len(ia), 2, generator=g, dtype=DT)
    pix_readme = -yb[:, :2] / yb[:, 2:] + noise
    pix_k = ref.point2pixel(yb, K) + 300 * noise
    out["pix_readme"], out["pix_k"] = pix_readme.numpy(), pix_k.numpy()
    for tag, Kt, pix in (("readme", None, pix_readme), ("k", K, pix_k)):
        for sname, smk in (("trustregion", lambda: ref.optim.strategy.TrustRegion()),
                           ("constant", lambda: ref.optim.strategy.Constant(damping=1e-4))):
            model = TwoPoseReproj(init.clone(), Kt)
            l, p, r = run(model, (pts, pix, ia, ib), smk(), 6)
            out[f"{tag}/{sname}/loss"], out[f"{tag}/{sname}/poses"], out[f"{tag}/{sname}/reject"] = l, p, r
            print(tag, sname, l, r)
    # a harder start (noise 0.15, small trust region) so that trials are rejected
    gh = torch.Generator().manual_seed(3)
    init_h = ref.se3(0.15 * torch.randn(N, 6, generator=gh, dtype=DT)).Exp() * gt
    out["poses0_hard"] = init_h.numpy()
    model = TwoPoseReproj(init_h.clone(), None)
    l, p, r = run(model, (pts, pix_readme, ia, ib), ref.optim.strategy.TrustRegion(radius=1e2), 8)
    out["hard/trustregion/loss"], out["hard/trustregion/poses"], out["hard/trustregion/reject"] = l, p, r
    print("hard", l, r)
    # bundle adjustment with intrinsics (README.md:163-198 sparse example + an extra op: point2pixel with K) on the inputs of
    # tests/golden/lm.npz "ba/*": not one of the fused families -> the generic block route (optim/blocks.py) must match
    g1 = np.load(os.path.join(os.path.dirname(OUT), "lm.npz"))
    T0, p0 = ref.SE3(torch.from_numpy(g1["ba/poses0"].copy())), torch.from_numpy(g1["ba/points0"].copy())
    cb, pb = torch.from_numpy(g1["ba/cidx"]), torch.from_numpy(g1["ba/pidx"])
    Kb = torch.tensor([[-1.2, 0.01, 0.05], [0.0, -0.9, -0.02], [0.0, 0.0, 1.0]], dtype=DT)
    pixb = torch.from_numpy(g1["ba/pix"].copy()) @ Kb[:2, :2].mT * 1.0 + Kb[:2, 2]

    class BAK(nn.Module):
        def __init__(self, poses, points):
            super().__init__()
            self.poses = ref.Parameter(poses)
            self.points_3d = nn.Parameter(points)

        def forward(self, observations, camera_indices, point_indices):
            y = self.poses[camera_indices].Act(self.points_3d[point_indices])
            return ref.point2pixel(y, Kb) - observations

    model = BAK(T0.clone(), p0.clone())
    opt = ref.optim.LM(model, strategy=ref.optim.strategy.TrustRegion())
    l, P, Q = [], [], []
    for _ in range(5):
        l.append(float(opt.step((pixb, cb, pb))))
        P.append(model.poses.detach().clone().numpy()); Q.append(model.points_3d.detach().clone().numpy())
    out["bak/K"], out["bak/pix"] = Kb.numpy(), pixb.numpy()
    out["bak/trustregion/loss"], out["bak/trustregion/poses"], out["bak/trustregion/points"] = np.array(l), np.stack(P), np.stack(Q)
    print("bak", l)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
