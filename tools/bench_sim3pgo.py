"""Time LM steps of Sim3 pose graphs (pp.module.PoseGraph with pp.Sim3 nodes) on seeded synthetic monocular-drift graphs of
1e4, 1e5 and 1e6 nodes with about 3 edges per node, on the fused route (optim/structured.py Sim3PGOProblem, one C call per
trial) and, where it fits, on the generic block route (optim/blocks.py BlockProblem) the same model takes when not
recognised.
    python tools/bench_sim3pgo.py [--nodes 10000,100000,1000000] [--steps 3] [--generic-max-nodes 100000]
Prints one JSON line per (size, dtype, route) with the card name and power limit read in the same run.  Times are
device-synchronised wall time per LM.step (all trials of the step); PCG iterations are those of the step's last solve.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pypose_b200 as pp  # noqa: E402
from pypose_b200.optim import blocks, structured  # noqa: E402
from pypose_b200.optim.solver import PCG  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        out = torch.cuda.get_device_name() + ", power limit unknown"
    return out


def problem(N, seed, dt):
    """An odometry chain whose relative scale drifts by 1e-3 per step, 2N loop closures between nodes 2-50 apart measured
    at unit scale, and a start chained from the drifted odometry with extra noise."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"

    def n(*s, sd=1.0):
        return torch.randn(*s, generator=g, device=dev, dtype=torch.float64) * sd
    steps = torch.zeros(N, 7, device=dev, dtype=torch.float64)
    steps[1:, 0] = 1.0
    steps[1:, 3:6] = n(N - 1, 3, sd=0.05)
    gt = pp.sim3(steps).Exp().cumprod(dim=0, left=False)
    a = torch.randint(0, N - 50, (2 * N,), generator=g, device=dev)
    loops = torch.stack([a, a + torch.randint(2, 50, (2 * N,), generator=g, device=dev)], 1)
    chain = torch.stack([torch.arange(N - 1, device=dev), torch.arange(1, N, device=dev)], 1)
    edges = torch.cat([chain, loops])
    E = edges.shape[0]
    noise = n(E, 7, sd=0.005)
    noise[: N - 1, 6] += 1e-3                                     # odometry scale drift
    Z = gt[edges[:, 0]].Inv() @ gt[edges[:, 1]] @ pp.sim3(noise).Exp()
    start = pp.sim3(n(N, 7, sd=0.02)).Exp() @ gt
    return pp.Sim3(start.tensor().to(dt)), (edges, pp.Sim3(Z.tensor().to(dt)))


def run(N, dt, route, steps, warmup):
    nodes, inp = problem(N, 0, dt)
    model = pp.module.PoseGraph(nodes)
    opt = pp.optim.LM(model, solver=PCG(tol=1e-4, maxiter=250), strategy=pp.optim.strategy.TrustRegion(), sparse=True)
    if route == "generic":
        params = [p for p in model.parameters() if p.requires_grad]
        opt._problem = blocks.BlockProblem.build(model, inp, params, structured._input_key(inp), None, None, opt.solver,
                                                 opt.model)
    times, iters, losses = [], [], []
    for s in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss = float(opt.step(inp))
        torch.cuda.synchronize()
        if s >= warmup:
            times.append(time.perf_counter() - t0)
            iters.append(getattr(opt._problem, "cg_iters", None))
            losses.append(loss)
    return {"nodes": N, "edges": int(inp[0].shape[0]), "dtype": str(dt).replace("torch.", ""),
            "route": type(opt._problem).__name__, "ms_per_step": [round(1e3 * t, 3) for t in times],
            "median_ms_per_step": round(1e3 * float(np.median(times)), 3), "pcg_iters": iters, "loss": losses}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", default="10000,100000,1000000")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--generic-max-nodes", type=int, default=100000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_sim3pgo.py measures on a CUDA device"
    gpu = card()
    for N in (int(v) for v in args.nodes.split(",")):
        for dt in (torch.float64, torch.float32):
            for route in ("fused", "generic"):
                if route == "generic" and N > args.generic_max_nodes:
                    continue
                try:
                    r = run(N, dt, route, args.steps, args.warmup)
                except torch.OutOfMemoryError:
                    r = {"nodes": N, "dtype": str(dt).replace("torch.", ""), "route": route, "error": "out of memory"}
                    torch.cuda.empty_cache()
                r["card"] = gpu
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
