"""Time LM steps of SO3 pose graphs (rotation averaging: pp.module.PoseGraph with pp.SO3 nodes) on seeded synthetic view
graphs, on the fused route (optim/structured.py SO3PGOProblem, one C call per trial) and, where it fits, on the generic
block route (optim/blocks.py BlockProblem) the same model takes when not recognised.  Two shapes, because the node-ordered
operator was shaped for about 6 slots per node and view graphs are much denser than SLAM graphs:
    sparse  1e4, 1e5 and 1e6 nodes at about 3 edges per node
    dense   1e4 nodes at about 40 edges per node, 1e5 at about 20
    python tools/bench_so3pgo.py [--shapes 10000x3,...] [--steps 3] [--generic-max-edges 400000]
Prints one JSON line per (shape, dtype, route) with the card name and power limit read in the same run.  Times are
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

SHAPES = "10000x3,100000x3,1000000x3,10000x40,100000x20"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        out = torch.cuda.get_device_name() + ", power limit unknown"
    return out


def problem(N, deg, seed, dt):
    """Random absolute rotations, a chain for connectivity plus (deg - 1) N random camera pairs (deg edges per node on
    average), relative rotations with 0.01 rad noise, and a start 0.1 rad from the truth."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"

    def n(*s, sd=1.0):
        return torch.randn(*s, generator=g, device=dev, dtype=torch.float64) * sd
    gt = pp.so3(n(N, 3)).Exp()
    M = (deg - 1) * N
    a = torch.randint(0, N, (M,), generator=g, device=dev)
    b = (a + torch.randint(1, N, (M,), generator=g, device=dev)) % N
    chain = torch.stack([torch.arange(N - 1, device=dev), torch.arange(1, N, device=dev)], 1)
    edges = torch.cat([chain, torch.stack([a, b], 1)])
    E = edges.shape[0]
    noise = n(E, 3, sd=0.01)
    Z = gt[edges[:, 0]].Inv() @ gt[edges[:, 1]] @ pp.so3(noise).Exp()
    start = pp.so3(n(N, 3, sd=0.1)).Exp() @ gt
    return pp.SO3(start.tensor().to(dt)), (edges, pp.SO3(Z.tensor().to(dt)))


def run(N, deg, dt, route, steps, warmup):
    nodes, inp = problem(N, deg, 0, dt)
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
    return {"nodes": N, "edges": int(inp[0].shape[0]), "edges_per_node": deg, "dtype": str(dt).replace("torch.", ""),
            "route": type(opt._problem).__name__, "ms_per_step": [round(1e3 * t, 3) for t in times],
            "median_ms_per_step": round(1e3 * float(np.median(times)), 3), "pcg_iters": iters, "loss": losses}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=SHAPES, help="comma-separated NODESxEDGES_PER_NODE")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--generic-max-edges", type=int, default=400000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_so3pgo.py measures on a CUDA device"
    gpu = card()
    for shape in args.shapes.split(","):
        N, deg = (int(v) for v in shape.split("x"))
        for dt in (torch.float64, torch.float32):
            for route in ("fused", "generic"):
                if route == "generic" and N * deg > args.generic_max_edges:
                    continue
                try:
                    r = run(N, deg, dt, route, args.steps, args.warmup)
                except torch.OutOfMemoryError:
                    r = {"nodes": N, "edges_per_node": deg, "dtype": str(dt).replace("torch.", ""), "route": route,
                         "error": "out of memory"}
                    torch.cuda.empty_cache()
                r["card"] = gpu
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
