"""Worker for tests/test_dist_nccl.py: the sharded LM on `world` GPUs (one process per GPU, NCCL for plumbing, NVLink
peer memory for the data path) — trajectories must equal the reference's single-process goldens; the peer all-reduce must
equal torch.distributed's."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{os.environ['MASTER_PORT']}", rank=rank, world_size=world,
                            device_id=dev)
    g = np.load(os.path.join(ROOT, "tests", "golden", "lm.npz"))
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    res = {}
    # ---- peer-memory all-reduce vs NCCL
    from pypose_b200._comm import PeerComm
    n = 100003
    comm = PeerComm.create(True, dev, 4 * ((n + 3) // 4 * 4 + 64) * 8 * 2 + 4096)
    res["peer_available"] = np.array([0 if comm is None else 1])
    if comm is not None:
        q = ((n + 3) // 4 + world - 1) // world * 4
        for dt in (torch.float32, torch.float64):
            for rep in range(3):
                t = torch.randn(n, dtype=dt, device=dev, generator=torch.Generator(device=dev).manual_seed(10 * rank + rep))
                ref = t.clone()
                dist.all_reduce(ref)
                comm.allreduce_(t, 0, 256 * ((world * q * 8 + 255) // 256))
                err = (t - ref).abs().max().item()
                assert err <= (1e-5 if dt == torch.float32 else 1e-13), (dt, err)
        comm.close()
    # ---- PoseInv: poses sharded; only the four scalar sums cross the GPUs
    P0, X = g["poseinv/P0"], g["poseinv/X"]
    lo, hi = rank * len(P0) // world, (rank + 1) * len(P0) // world
    net = InvNet(pp.SE3(cu(P0[lo:hi])))
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), group=True)
    Xs = pp.SE3(cu(X[lo:hi]))
    losses = [float(opt.step(Xs)) for _ in range(4)]
    res["poseinv_peer"] = np.array([int(getattr(opt._problem, "_ds", None) is not None and opt._problem._ds.comm is not None)])
    gathered = [torch.zeros(len(P0) // world, 7, dtype=torch.float64, device=dev) for _ in range(world)]
    dist.all_gather(gathered, net.pose.detach().tensor().contiguous())
    res["poseinv_loss"], res["poseinv_poses"] = np.array(losses), torch.cat(gathered).cpu().numpy()
    # ---- Reproj: observations sharded, poses replicated
    # both exchange forms of the sharded reprojection trial (optim/_lmstep.py reproj_gather): owner = reduce-scatter of the
    # blocks + all-gather of the trial poses, gather = every rank receives all blocks and solves every camera
    # ... and both splits: rows as stored (every rank holds rows of every camera) and rows sorted by camera before the
    # split (SURVEY.md §8e: a rank then holds a subset of the cameras; the `present` mask / local camera list route)
    # the size rule is pinned to one form, the same on every rank: a limit of 0 picks owner, one above every payload gather
    from pypose_b200.optim import _lmstep
    gather_bytes = _lmstep.GATHER_BYTES
    for form, split, case, steps in [(f, sp, c, n) for f in ("owner", "gather") for sp in ("stored", "sorted")
                                     for c, n in (("reproj", 4), ("reproj_hard", 6))]:
        _lmstep.GATHER_BYTES = 1 << 62 if form == "gather" else 0
        tag = case + ("_gather" if form == "gather" else "") + ("_sorted" if split == "sorted" else "")
        pts, pix, cidx = g[f"{case}/pts"], g[f"{case}/pix"], g[f"{case}/cidx"]
        if split == "sorted":
            order = np.argsort(cidx, kind="stable")
            pts, pix, cidx = pts[order], pix[order], cidx[order]
        M = len(cidx)
        sl = slice(rank * M // world, (rank + 1) * M // world)
        net2 = pp.module.PoseReproj(pp.SE3(cu(g[f"{case}/poses0"])))
        opt2 = pp.optim.LM(net2, strategy=pp.optim.strategy.TrustRegion(), group=True)
        inp = (cu(pts[sl]), cu(pix[sl]), cu(cidx[sl]))
        l2, rej = [], []
        for _ in range(steps):
            l2.append(float(opt2.step(inp)))
            rej.append(opt2.reject_count)
        res[f"{tag}_peer"] = np.array([int(getattr(opt2._problem, "_ds", None) is not None and opt2._problem._ds.comm is not None)])
        res[f"{tag}_loss"], res[f"{tag}_poses"], res[f"{tag}_reject"] = np.array(l2), net2.poses.detach().cpu().numpy(), np.array(rej)
        # every rank holds the same poses bit for bit
        mine = net2.poses.detach().tensor().contiguous()
        other = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(other, mine)
        assert all(torch.equal(o, mine) for o in other), "replicated poses diverged between ranks"
    _lmstep.GATHER_BYTES = gather_bytes
    # ---- PGO: edges sharded, nodes replicated
    edges, Z = g["pgo/edges"], g["pgo/Z"]
    E = len(edges)
    sl = slice(rank * E // world, (rank + 1) * E // world)
    net3 = pp.module.PoseGraph(pp.SE3(cu(g["pgo/nodes0"])))
    opt3 = pp.optim.LM(net3, strategy=pp.optim.strategy.TrustRegion(), solver=pp.optim.solver.PCG(tol=1e-12), sparse=True,
                       group=True)
    inp3 = (cu(edges[sl]), pp.SE3(cu(Z[sl])))
    res["pgo_loss"] = np.array([float(opt3.step(inp3)) for _ in range(5)])
    res["pgo_poses"] = net3.nodes.detach().cpu().numpy()
    # ---- BA: observations sharded, poses and points replicated
    pixb, cb, pb = g["ba/pix"], g["ba/cidx"], g["ba/pidx"]
    Mb = len(cb)
    sl = slice(rank * Mb // world, (rank + 1) * Mb // world)
    net4 = pp.module.BundleAdjustment(pp.SE3(cu(g["ba/poses0"])), cu(g["ba/points0"]))
    opt4 = pp.optim.LM(net4, strategy=pp.optim.strategy.TrustRegion(), solver=pp.optim.solver.PCG(tol=1e-12), sparse=True,
                       group=True)
    inp4 = (cu(pixb[sl]), cu(cb[sl]), cu(pb[sl]))
    res["ba_loss"] = np.array([float(opt4.step(inp4)) for _ in range(5)])
    res["ba_poses"], res["ba_points"] = net4.poses.detach().cpu().numpy(), net4.points_3d.detach().cpu().numpy()
    if rank == 0:
        np.savez(out, **res)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
