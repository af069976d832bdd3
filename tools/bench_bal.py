"""Time LM steps of BAL bundle adjustment (pp.module.BALBundleAdjustment) on seeded synthetic problems of the sizes of
three public BAL files, on the fused route (optim/structured.py BALProblem, csrc/bal.cu) and, where it finishes in
reasonable time, on the generic block route (optim/blocks.py BlockProblem) the same model takes when not recognised.

    python tools/bench_bal.py [--sizes trafalgar,ladybug,venice] [--steps 3] [--generic-max-obs 1000000]

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

SIZES = {  # cameras, points, observations
    "trafalgar": (257, 65132, 225911),
    "ladybug": (1723, 156502, 678718),
    "venice": (1778, 993923, 5001946),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        out = torch.cuda.get_device_name() + ", power limit unknown"
    return out


def problem(C, P, M, seed, dt):
    """Seeded BAL-like problem on the GPU: cameras looking down -z at points 3-8 units away, f ~ 500, |k1| <= 0.1,
    every point seen by two cameras, observations with 0.5 px noise, and a perturbed start."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"

    def n(*s, sd=1.0):
        return torch.randn(*s, generator=g, device=dev, dtype=torch.float64) * sd

    T = pp.se3(torch.cat([n(C, 3, sd=0.3), n(C, 3, sd=0.05)], 1)).Exp()
    pc = torch.cat([(torch.rand(P, 2, generator=g, device=dev, dtype=torch.float64) - 0.5) * 3,
                    -(3 + 5 * torch.rand(P, 1, generator=g, device=dev, dtype=torch.float64))], 1)
    pw = pp.SE3(T[:1].Inv().tensor().expand(P, 7)).Act(pc)      # camera 0's frame -> world
    K = torch.stack([450 + 100 * torch.rand(C, generator=g, device=dev, dtype=torch.float64),
                     (torch.rand(C, generator=g, device=dev, dtype=torch.float64) - 0.5) * 0.2,
                     (torch.rand(C, generator=g, device=dev, dtype=torch.float64) - 0.5) * 0.02], 1)
    c2 = torch.randint(0, C, (P,), generator=g, device=dev)
    c3 = (c2 + 1 + torch.randint(0, C - 1, (P,), generator=g, device=dev)) % C
    cidx = torch.cat([c2, c3, torch.randint(0, C, (M - 2 * P,), generator=g, device=dev)])
    pidx = torch.cat([torch.arange(P, device=dev), torch.arange(P, device=dev),
                      torch.randint(0, P, (M - 2 * P,), generator=g, device=dev)])
    true = pp.module.BALBundleAdjustment(K, T, pw)
    with torch.no_grad():
        pix = true(torch.zeros(M, 2, device=dev, dtype=torch.float64), cidx, pidx) + n(M, 2, sd=0.5)
    T0 = (pp.se3(torch.cat([n(C, 3, sd=0.02), n(C, 3, sd=0.005)], 1)).Exp() * T)
    K0 = K * torch.tensor([1.01, 1.0, 1.0], device=dev, dtype=torch.float64)
    P0 = pw + n(P, 3, sd=0.05)
    return (K0.to(dt), pp.SE3(T0.tensor().to(dt)), P0.to(dt)), (pix.to(dt), cidx, pidx)


def run(name, dt, route, steps, warmup):
    C, P, M = SIZES[name]
    (K0, T0, P0), inp = problem(C, P, M, 0, dt)
    model = pp.module.BALBundleAdjustment(K0, T0, P0)
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
    return {"size": name, "cameras": C, "points": P, "observations": M, "dtype": str(dt).replace("torch.", ""),
            "route": type(opt._problem).__name__, "ms_per_step": [round(1e3 * t, 3) for t in times],
            "median_ms_per_step": round(1e3 * float(np.median(times)), 3), "pcg_iters": iters, "loss": losses}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="trafalgar,ladybug,venice")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--generic-max-obs", type=int, default=300000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_bal.py measures on a CUDA device"
    gpu = card()
    for name in args.sizes.split(","):
        for dt in (torch.float64, torch.float32):
            for route in ("fused", "generic"):
                if route == "generic" and SIZES[name][2] > args.generic_max_obs:
                    continue
                r = run(name, dt, route, args.steps, args.warmup)
                r["card"] = gpu
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
