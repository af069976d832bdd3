"""Worker for tests/test_dist_gloo.py: runs the sharded LM on `world` CPU processes (gloo) with the
oracle-backed test kernels and writes its loss / pose trajectory to an .npz."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tests.conftest  # noqa: F401,E402  (installs the CPU oracle kernels)
import pypose_b200 as pp  # noqa: E402
from torch import nn  # noqa: E402


class InvNet(nn.Module):
    def __init__(self, pose):
        super().__init__()
        self.pose = pp.Parameter(pose)

    def forward(self, input):
        return (self.pose @ input).Log().tensor()


def main():
    out = sys.argv[1]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{os.environ['MASTER_PORT']}", rank=rank, world_size=world)
    g = np.load(os.path.join(ROOT, "tests", "golden", "lm.npz"))
    res = {}
    # PoseInv: poses sharded (each rank owns a slice); scalar sums all-reduced
    P0, X = g["poseinv/P0"], g["poseinv/X"]
    lo, hi = rank * len(P0) // world, (rank + 1) * len(P0) // world
    net = InvNet(pp.SE3(torch.from_numpy(P0[lo:hi].copy())))
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), group=True)
    Xs = pp.SE3(torch.from_numpy(X[lo:hi].copy()))
    losses = [float(opt.step(Xs)) for _ in range(4)]
    gathered = [torch.zeros(len(P0) // world, 7, dtype=torch.float64) for _ in range(world)]
    dist.all_gather(gathered, net.pose.detach().tensor().contiguous())
    res["poseinv_loss"], res["poseinv_poses"] = np.array(losses), torch.cat(gathered).numpy()
    # Reproj: residuals sharded, poses replicated; [H | g] and the scalars all-reduced
    for case, steps in (("reproj", 4), ("reproj_hard", 6)):
        pts, pix, cidx = g[f"{case}/pts"], g[f"{case}/pix"], g[f"{case}/cidx"]
        M = len(cidx)
        sl = slice(rank * M // world, (rank + 1) * M // world)
        net2 = pp.module.PoseReproj(pp.SE3(torch.from_numpy(g[f"{case}/poses0"].copy())))
        opt2 = pp.optim.LM(net2, strategy=pp.optim.strategy.TrustRegion(), group=True)
        inp = (torch.from_numpy(pts[sl]), torch.from_numpy(pix[sl]), torch.from_numpy(cidx[sl]))
        l2, rej = [], []
        for _ in range(steps):
            l2.append(float(opt2.step(inp)))
            rej.append(opt2.reject_count)
        res[f"{case}_loss"], res[f"{case}_poses"], res[f"{case}_reject"] = np.array(l2), net2.poses.detach().numpy(), np.array(rej)
    # PGO: edges sharded, nodes replicated; Hd | g, every PCG matvec and the scalars all-reduced
    edges, Z = g["pgo/edges"], g["pgo/Z"]
    E = len(edges)
    sl = slice(rank * E // world, (rank + 1) * E // world)
    net3 = pp.module.PoseGraph(pp.SE3(torch.from_numpy(g["pgo/nodes0"].copy())))
    opt3 = pp.optim.LM(net3, strategy=pp.optim.strategy.TrustRegion(), solver=pp.optim.solver.PCG(tol=1e-12), sparse=True,
                       group=True)
    inp3 = (torch.from_numpy(edges[sl]), pp.SE3(torch.from_numpy(Z[sl].copy())))
    res["pgo_loss"] = np.array([float(opt3.step(inp3)) for _ in range(5)])
    res["pgo_poses"] = net3.nodes.detach().numpy()
    # BA: observations sharded, poses and points replicated
    pixb, cb, pb = g["ba/pix"], g["ba/cidx"], g["ba/pidx"]
    Mb = len(cb)
    sl = slice(rank * Mb // world, (rank + 1) * Mb // world)
    net4 = pp.module.BundleAdjustment(pp.SE3(torch.from_numpy(g["ba/poses0"].copy())), torch.from_numpy(g["ba/points0"].copy()))
    opt4 = pp.optim.LM(net4, strategy=pp.optim.strategy.TrustRegion(), solver=pp.optim.solver.PCG(tol=1e-12), sparse=True,
                       group=True)
    inp4 = (torch.from_numpy(pixb[sl]), torch.from_numpy(cb[sl]), torch.from_numpy(pb[sl]))
    res["ba_loss"] = np.array([float(opt4.step(inp4)) for _ in range(5)])
    res["ba_poses"], res["ba_points"] = net4.poses.detach().numpy(), net4.points_3d.detach().numpy()
    # ---- bench_legs._all_continue: ranks that want a different number of timed regions run the same number (the sharded
    # legs exchange data inside a step; the first 2-GPU bench of round 2 deadlocked on ranks falling out of step)
    import bench_legs
    bench_legs._WORLD["size"], bench_legs._WORLD["dev"] = world, "cpu"
    wanted, ran = 5 + 4 * rank, 0
    while bench_legs._all_continue(ran < wanted):
        ran += 1
    # ---- optim/_lmstep.py: host side of the sharded reprojection exchange (which rank holds rows of which camera; sizes of
    # the two exchange forms)
    from types import SimpleNamespace
    from pypose_b200.optim import _lmstep
    C = 7
    rows = {0: [3, 0, 2, 0, 0, 1, 0], 1: [0, 0, 4, 5, 0, 0, 0]}[rank]
    seg = torch.tensor(np.concatenate([[0], np.cumsum(rows)]), dtype=torch.int32)
    present, cams = _lmstep._present_mask(SimpleNamespace(seg=seg, group=True), SimpleNamespace(world=world))
    res["present"], res["cams"] = present.numpy(), cams.numpy()
    res["payload_gather"] = np.array(_lmstep.reproj_payload(1000, 2, 4))
    gather_bytes, _lmstep.GATHER_BYTES = _lmstep.GATHER_BYTES, 0      # owner form at any size, on every rank
    try:
        res["payload_owner"] = np.array(_lmstep.reproj_payload(1000, 2, 4))
    finally:
        _lmstep.GATHER_BYTES = gather_bytes
    counts = [torch.zeros(1, dtype=torch.int64) for _ in range(world)]
    dist.all_gather(counts, torch.tensor([ran]))
    res["regions_run"] = torch.cat(counts).numpy()
    if rank == 0:
        np.savez(out, **res)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
