"""Record LM trajectories from the REFERENCE's own optimizer (pypose v0.9.5, fp64, CPU):

    python oracle/make_golden_lm.py        # writes tests/golden/lm.npz

* PoseInv: README.md:120-135 InvNet, N = 6 poses, 4 steps, Constant(1e-4) and default TrustRegion.
* Reproj:  r = -(T_c p)[:2]/(T_c p)[2] - z with C = 4 cameras / 40 observations, 4 steps, Constant(1e-4).
"""
import os
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "lm.npz")


class InvNet(nn.Module):
    def __init__(self, pose):
        super().__init__()
        self.pose = ref.Parameter(pose)

    def forward(self, input):
        return (self.pose @ input).Log().tensor()


class Reproj(nn.Module):
    def __init__(self, poses):
        super().__init__()
        self.poses = ref.Parameter(poses)

    def forward(self, points, pixels, cidx):
        y = self.poses[cidx].Act(points)
        return -y[..., :2] / y[..., 2:] - pixels


class PoseGraph(nn.Module):                 # examples/module/pgo/pgo.py:15-25
    def __init__(self, nodes):
        super().__init__()
        self.nodes = ref.Parameter(nodes)

    def forward(self, edges, poses):
        node1 = self.nodes[edges[..., 0]]
        node2 = self.nodes[edges[..., 1]]
        return (poses.Inv() @ node1.Inv() @ node2).Log().tensor()


class BA(nn.Module):                        # README.md:163-198 (without the bae-only sjac / psjac markers)
    def __init__(self, poses, points_3d):
        super().__init__()
        self.poses = ref.Parameter(poses)
        self.points_3d = ref.Parameter(points_3d)

    def forward(self, observations, camera_indices, point_indices):
        pts = self.poses[camera_indices].Act(self.points_3d[point_indices])
        return -pts[..., :2] / pts[..., 2].unsqueeze(-1) - observations


def run(model, input, strategy, steps, pname):
    opt = ref.optim.LM(model, strategy=strategy)
    losses, poses, rejects = [], [], []
    for _ in range(steps):
        losses.append(float(opt.step(input)))
        poses.append(getattr(model, pname).detach().clone().numpy())
        rejects.append(opt.reject_count)
    return np.array(losses), np.stack(poses), np.array(rejects)


def main():
    torch.manual_seed(7)
    g = {}
    P0 = ref.randn_SE3(6, sigma=0.3, dtype=torch.float64)
    X = ref.randn_SE3(6, sigma=0.8, dtype=torch.float64)
    g["poseinv/P0"], g["poseinv/X"] = P0.numpy().copy(), X.numpy().copy()
    for name, strat in (("constant", lambda: ref.optim.strategy.Constant(damping=1e-4)),
                        ("trustregion", lambda: ref.optim.strategy.TrustRegion()),
                        ("adaptive", lambda: ref.optim.strategy.Adaptive(damping=1e-2))):
        losses, poses, rej = run(InvNet(P0.clone()), X, strat(), 4, "pose")
        g[f"poseinv/{name}/loss"], g[f"poseinv/{name}/poses"], g[f"poseinv/{name}/reject"] = losses, poses, rej

    C, M = 4, 40
    gt = ref.randn_SE3(C, sigma=0.2, dtype=torch.float64)
    gt.tensor()[:, 2] += 0.0
    cidx = torch.arange(M) % C
    pts_cam = torch.rand(M, 3, dtype=torch.float64) * torch.tensor([4.0, 4.0, 4.0]) + torch.tensor([-2.0, -2.0, 2.0])
    pts = gt[cidx].Inv().Act(pts_cam)                       # world points seen at pts_cam in the GT cameras
    pix = -pts_cam[:, :2] / pts_cam[:, 2:] + 1e-3 * torch.randn(M, 2, dtype=torch.float64)
    init = ref.se3(0.05 * torch.randn(C, 6, dtype=torch.float64)).Exp() * gt
    g["reproj/poses0"], g["reproj/pts"], g["reproj/pix"], g["reproj/cidx"] = (init.numpy().copy(), pts.numpy().copy(),
                                                                               pix.numpy().copy(), cidx.numpy().copy())
    for name, strat in (("constant", lambda: ref.optim.strategy.Constant(damping=1e-4)),
                        ("trustregion", lambda: ref.optim.strategy.TrustRegion())):
        losses, poses, rej = run(Reproj(init.clone()), (pts, pix, cidx), strat(), 4, "poses")
        g[f"reproj/{name}/loss"], g[f"reproj/{name}/poses"], g[f"reproj/{name}/reject"] = losses, poses, rej
    # a badly initialised problem whose default TrustRegion run rejects steps (reject counts 4,0,0,1,0,0):
    # exercises the cumulative damping / undo path of optimizer.py:662-680
    torch.manual_seed(0)
    gt = ref.randn_SE3(C, sigma=0.2, dtype=torch.float64)
    pts_cam = torch.rand(M, 3, dtype=torch.float64) * 4 + torch.tensor([-2.0, -2.0, 2.0])
    pts = gt[cidx].Inv().Act(pts_cam)
    pix = -pts_cam[:, :2] / pts_cam[:, 2:]
    init = ref.se3(0.8 * torch.randn(C, 6, dtype=torch.float64)).Exp() * gt
    g["reproj_hard/poses0"], g["reproj_hard/pts"], g["reproj_hard/pix"], g["reproj_hard/cidx"] = (
        init.numpy().copy(), pts.numpy().copy(), pix.numpy().copy(), cidx.numpy().copy())
    losses, poses, rej = run(Reproj(init.clone()), (pts, pix, cidx), ref.optim.strategy.TrustRegion(), 6, "poses")
    g["reproj_hard/trustregion/loss"], g["reproj_hard/trustregion/poses"], g["reproj_hard/trustregion/reject"] = losses, poses, rej
    # pose graph: 10 nodes on a noisy loop, odometry + loop-closure edges, dense reference LM (Cholesky)
    torch.manual_seed(21)
    N = 10
    gtn = ref.se3(torch.cat([torch.tensor([[1.0, 0.2, 0.0, 0.0, 0.0, 0.35]], dtype=torch.float64)] * N)).Exp().cumprod(dim=0, left=False)
    pairs = [(i, i + 1) for i in range(N - 1)] + [(0, 5), (2, 7), (3, 9), (1, 8), (9, 0)]
    edges = torch.tensor(pairs)
    Zm = gtn[edges[:, 0]].Inv() @ gtn[edges[:, 1]]
    Zm = ref.se3(0.02 * torch.randn(len(pairs), 6, dtype=torch.float64)).Exp() @ Zm
    init = ref.se3(0.15 * torch.randn(N, 6, dtype=torch.float64)).Exp() @ gtn
    g["pgo/nodes0"], g["pgo/edges"], g["pgo/Z"] = init.numpy().copy(), edges.numpy().copy(), Zm.numpy().copy()
    for name, strat in (("trustregion", lambda: ref.optim.strategy.TrustRegion()),
                        ("constant", lambda: ref.optim.strategy.Constant(damping=1e-4))):
        losses, poses, rej = run(PoseGraph(init.clone()), (edges, Zm), strat(), 5, "nodes")
        g[f"pgo/{name}/loss"], g[f"pgo/{name}/poses"], g[f"pgo/{name}/reject"] = losses, poses, rej

    # bundle adjustment: 5 cameras x 16 points, every point seen by 3 cameras, poses AND points optimised
    torch.manual_seed(31)
    Cb, Pb = 5, 16
    gtb = ref.randn_SE3(Cb, sigma=0.15, dtype=torch.float64)
    ptsw = torch.rand(Pb, 3, dtype=torch.float64) * torch.tensor([4.0, 4.0, 3.0]) + torch.tensor([-2.0, -2.0, 3.0])
    cb = torch.tensor([(j + o) % Cb for j in range(Pb) for o in range(3)])
    pb = torch.tensor([j for j in range(Pb) for _ in range(3)])
    yb = gtb[cb].Act(ptsw[pb])
    pixb = -yb[:, :2] / yb[:, 2:] + 1e-3 * torch.randn(len(cb), 2, dtype=torch.float64)
    poses0 = ref.se3(0.03 * torch.randn(Cb, 6, dtype=torch.float64)).Exp() * gtb
    pts0 = ptsw + 0.05 * torch.randn(Pb, 3, dtype=torch.float64)
    g["ba/poses0"], g["ba/points0"], g["ba/pix"], g["ba/cidx"], g["ba/pidx"] = (poses0.numpy().copy(), pts0.numpy().copy(),
                                                                                pixb.numpy().copy(), cb.numpy().copy(), pb.numpy().copy())
    for name, strat in (("trustregion", lambda: ref.optim.strategy.TrustRegion()),
                        ("constant", lambda: ref.optim.strategy.Constant(damping=1e-4))):
        model = BA(poses0.clone(), pts0.clone())
        opt = ref.optim.LM(model, strategy=strat())
        losses, ps, qs, rej = [], [], [], []
        for _ in range(5):
            losses.append(float(opt.step((pixb, cb, pb))))
            ps.append(model.poses.detach().clone().numpy()); qs.append(model.points_3d.detach().clone().numpy())
            rej.append(opt.reject_count)
        g[f"ba/{name}/loss"], g[f"ba/{name}/poses"], g[f"ba/{name}/points"], g[f"ba/{name}/reject"] = (
            np.array(losses), np.stack(ps), np.stack(qs), np.array(rej))

    # robust kernels (default FastTriggs corrector): reprojection with 10 % gross outliers under Huber,
    # PoseInv under Cauchy (optimizer.py:474-480, corrector.py:73-95, kernel.py)
    torch.manual_seed(3)
    gt = ref.randn_SE3(C, sigma=0.2, dtype=torch.float64)
    pts_cam = torch.rand(M, 3, dtype=torch.float64) * 4 + torch.tensor([-2.0, -2.0, 2.0])
    pts = gt[cidx].Inv().Act(pts_cam)
    pix = -pts_cam[:, :2] / pts_cam[:, 2:]
    pix[::10] += 0.5 * torch.randn(M // 10, 2, dtype=torch.float64)
    init = ref.se3(0.05 * torch.randn(C, 6, dtype=torch.float64)).Exp() * gt
    g["robust_reproj/poses0"], g["robust_reproj/pts"], g["robust_reproj/pix"], g["robust_reproj/cidx"] = (
        init.numpy().copy(), pts.numpy().copy(), pix.numpy().copy(), cidx.numpy().copy())
    for kname, kern in (("huber", lambda: ref.optim.kernel.Huber(delta=0.05)), ("cauchy", lambda: ref.optim.kernel.Cauchy(delta=0.1)),
                        ("pseudohuber", lambda: ref.optim.kernel.PseudoHuber(delta=0.05)),
                        ("softlone", lambda: ref.optim.kernel.SoftLOne(delta=0.1)), ("arctan", lambda: ref.optim.kernel.Arctan(delta=0.3))):
        model = Reproj(init.clone())
        opt = ref.optim.LM(model, strategy=ref.optim.strategy.TrustRegion(), kernel=kern())
        losses, poses, rej = [], [], []
        for _ in range(5):
            losses.append(float(opt.step((pts, pix, cidx))))
            poses.append(model.poses.detach().clone().numpy()); rej.append(opt.reject_count)
        g[f"robust_reproj/{kname}/loss"], g[f"robust_reproj/{kname}/poses"], g[f"robust_reproj/{kname}/reject"] = (
            np.array(losses), np.stack(poses), np.array(rej))
    net = InvNet(P0.clone())
    opt = ref.optim.LM(net, strategy=ref.optim.strategy.Constant(damping=1e-4), kernel=ref.optim.kernel.Cauchy(delta=0.5))
    losses, poses = [], []
    for _ in range(4):
        losses.append(float(opt.step(X))); poses.append(net.pose.detach().clone().numpy())
    g["poseinv/cauchy/loss"], g["poseinv/cauchy/poses"] = np.array(losses), np.stack(poses)
    # pose graph with information matrices (examples/module/pgo/pgo.py:75: optimizer.step(input, weight=infos)):
    # per-edge SPD (E,6,6) and one shared (6,6)
    torch.manual_seed(77)
    edges_t, Z_t = torch.from_numpy(g["pgo/edges"]), ref.SE3(torch.from_numpy(g["pgo/Z"].copy()))
    Bw = torch.randn(edges_t.shape[0], 6, 6, dtype=torch.float64)
    infos = Bw @ Bw.mT / 6 + 0.5 * torch.eye(6, dtype=torch.float64)
    g["pgo_w/infos"] = infos.numpy().copy()
    for name, strat, W in (("trustregion", lambda: ref.optim.strategy.TrustRegion(), infos),
                           ("constant", lambda: ref.optim.strategy.Constant(damping=1e-4), infos),
                           ("shared", lambda: ref.optim.strategy.TrustRegion(), infos[3])):
        model = PoseGraph(ref.SE3(torch.from_numpy(g["pgo/nodes0"].copy())))
        opt = ref.optim.LM(model, strategy=strat())
        losses, poses, rej = [], [], []
        for _ in range(5):
            losses.append(float(opt.step((edges_t, Z_t), weight=W)))
            poses.append(model.nodes.detach().clone().numpy()); rej.append(opt.reject_count)
        g[f"pgo_w/{name}/loss"], g[f"pgo_w/{name}/poses"], g[f"pgo_w/{name}/reject"] = np.array(losses), np.stack(poses), np.array(rej)
    # robust kernels on the block-sparse families: pose graph with outlier edges and bundle adjustment with outlier pixels
    # (reference: dense LM, kernel + default FastTriggs corrector, TrustRegion)
    torch.manual_seed(88)
    Zo = Z_t.tensor().clone()
    Zo[::4] = (ref.se3(0.4 * torch.randn(Zo[::4].shape[0], 6, dtype=torch.float64)).Exp() @ ref.SE3(Zo[::4])).tensor()
    g["pgo_robust/Z"] = Zo.numpy().copy()
    for kname, kern in (("huber", lambda: ref.optim.kernel.Huber(delta=0.1)), ("cauchy", lambda: ref.optim.kernel.Cauchy(delta=0.2))):
        model = PoseGraph(ref.SE3(torch.from_numpy(g["pgo/nodes0"].copy())))
        opt = ref.optim.LM(model, strategy=ref.optim.strategy.TrustRegion(), kernel=kern())
        losses, poses, rej = [], [], []
        for _ in range(5):
            losses.append(float(opt.step((edges_t, ref.SE3(Zo)))))
            poses.append(model.nodes.detach().clone().numpy()); rej.append(opt.reject_count)
        g[f"pgo_robust/{kname}/loss"], g[f"pgo_robust/{kname}/poses"], g[f"pgo_robust/{kname}/reject"] = np.array(losses), np.stack(poses), np.array(rej)
    pixo = torch.from_numpy(g["ba/pix"].copy())
    pixo[::7] += 0.3 * torch.randn(pixo[::7].shape, dtype=torch.float64)
    g["ba_robust/pix"] = pixo.numpy().copy()
    cb_t, pb_t = torch.from_numpy(g["ba/cidx"]), torch.from_numpy(g["ba/pidx"])
    for kname, kern in (("huber", lambda: ref.optim.kernel.Huber(delta=0.05)),):
        model = BA(ref.SE3(torch.from_numpy(g["ba/poses0"].copy())), torch.from_numpy(g["ba/points0"].copy()))
        opt = ref.optim.LM(model, strategy=ref.optim.strategy.TrustRegion(), kernel=kern())
        losses, poses, points, rej = [], [], [], []
        for _ in range(5):
            losses.append(float(opt.step((pixo, cb_t, pb_t))))
            poses.append(model.poses.detach().clone().numpy()); points.append(model.points_3d.detach().clone().numpy())
            rej.append(opt.reject_count)
        g[f"ba_robust/{kname}/loss"], g[f"ba_robust/{kname}/poses"] = np.array(losses), np.stack(poses)
        g[f"ba_robust/{kname}/points"], g[f"ba_robust/{kname}/reject"] = np.stack(points), np.array(rej)
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, {k: (v if v.ndim == 1 and v.size <= 4 else v.shape) for k, v in g.items() if "loss" in k or "reject" in k})


if __name__ == "__main__":
    main()
