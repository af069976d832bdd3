"""Time pp.metric.ape / rpe end to end per call (host reads included) at 1e5, 1e6 and 1e7 poses, the distance walk on
its own, and the reference formulation (dense time-difference matrix, per-pose Python lists) in eager torch on the same
GPU where it fits.  Prints the card and its power limit, then one JSON line per measurement.

    python tools/bench_metric.py [--sizes 1e5,1e6,1e7] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pypose_b200 as pp  # noqa: E402
from pypose_b200.metric import ape_rpe as A  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def traj(n, dev, g):
    step = torch.randn(n, 3, device=dev, dtype=torch.float64, generator=g) * 0.05 + 0.02
    step[(torch.arange(n, device=dev) // 5) % 4 == 0] = 0.0        # stationary runs
    q = torch.randn(n, 4, device=dev, dtype=torch.float64, generator=g) * 0.1
    q[:, 3] += 1.0
    return pp.SE3(torch.cat([torch.cumsum(step, 0), q / q.norm(dim=-1, keepdim=True)], -1))


def timed(f, reps):
    f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    return ts[len(ts) // 2]


def ref_associate(rs, es, diff=0.01):
    """The reference's association: the full (N_short, N_long) matrix, min over it, lists."""
    short, long_ = (rs, es) if len(es) > len(rs) else (es, rs)
    v, j = (short[:, None] - long_[None]).abs().min(dim=-1)
    i = torch.arange(len(short), device=rs.device)
    return i[v < diff].tolist(), j[v < diff].tolist()


def ref_ape(rs, rp, es, ep):
    i, j = ref_associate(rs, es)
    e = (ep[j].translation() - rp[i].translation()).norm(dim=-1)
    return [torch.max(e), torch.min(e), e.mean(), e.median(), e.square().mean().sqrt(), e.square().sum(), e.std()]


def ref_rpe_frame(rs, rp, es, ep):
    i, j = ref_associate(rs, es)
    r, e = rp[i], ep[j]
    ids = torch.arange(0, len(i), 1, device=rs.device)
    a, b = ids[:-1].tolist(), ids[1:].tolist()
    E = (r[a].Inv() @ r[b]).Inv() @ (e[a].Inv() @ e[b])
    err = E.translation().norm(dim=-1)
    return [torch.max(err), torch.min(err), err.mean(), err.median()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1e5,1e6,1e7")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-size", type=int, default=20000)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    print("card:", card(), flush=True)
    for n in [int(float(s)) for s in a.sizes.split(",")]:
        rp, ep = traj(n, dev, g), traj(n, dev, g)
        rs = torch.arange(n, device=dev, dtype=torch.float64) * 0.01
        es = rs + 0.001
        runs = {
            "ape": lambda: pp.metric.ape(rs, rp, es, ep),
            "ape_align_scale": lambda: pp.metric.ape(rs, rp, es, ep, align=True, scale=True),
            "rpe_frame": lambda: pp.metric.rpe(rs, rp, es, ep),
            "rpe_distance": lambda: pp.metric.rpe(rs, rp, es, ep, associate="distance", delta=1.0),
            "rpe_distance_all": lambda: pp.metric.rpe(rs, rp, es, ep, associate="distance", delta=1.0, all=True),
        }
        for k, f in runs.items():
            print(json.dumps({"what": k, "poses": n, "ms": round(1e3 * timed(f, a.reps), 3)}), flush=True)
        idx = torch.arange(n, device=dev)
        t = timed(lambda: A._pairs_by_dist(ep.tensor(), idx, None, 1.0, 0.1, False), a.reps)
        print(json.dumps({"what": "walk (pairs_dist all=False: walk kernel + one host read)", "poses": n,
                          "ms": round(1e3 * t, 3), "ns_per_pose": round(1e9 * t / n, 2)}), flush=True)
        del rp, ep, rs, es
        torch.cuda.empty_cache()
    n = a.ref_size
    rp, ep = traj(n, dev, g), traj(n, dev, g)
    rs = torch.arange(n, device=dev, dtype=torch.float64) * 0.01
    es = rs + 0.001
    for k, f, o in (("ape", ref_ape, lambda: pp.metric.ape(rs, rp, es, ep)),
                    ("rpe_frame", ref_rpe_frame, lambda: pp.metric.rpe(rs, rp, es, ep))):
        print(json.dumps({"what": f"reference formulation {k}", "poses": n,
                          "ms": round(1e3 * timed(lambda: f(rs, rp, es, ep), a.reps), 3),
                          "this_ms": round(1e3 * timed(o, a.reps), 3)}), flush=True)


if __name__ == "__main__":
    main()
