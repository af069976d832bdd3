"""Time pp.module.LQR on an LTI system: the CUDA route (csrc/lqr.cu) against the generic route (the reference's algorithm in
torch ops) on the same GPU, forward and forward+backward, fp32 and fp64.  Prints problem-steps/s (B * T / time).  The
time-invariant case reads A, B, Q, p from one copy and moves almost no HBM bytes, so it is latency-bound.
Usage: python tools/bench_lqr.py [--quick]"""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pypose_b200 as pp  # noqa: E402


def problem(nb, T, ns, nc, dtype, dev):
    g = torch.Generator(device="cpu").manual_seed(0)
    n = ns + nc
    M = torch.randn(n, n, generator=g, dtype=dtype)
    Q = (M.mT @ M + torch.eye(n, dtype=dtype)).to(dev).expand(nb, n, n).requires_grad_()
    p = torch.randn(nb, n, generator=g, dtype=dtype).to(dev).requires_grad_()
    A = (0.8 * torch.eye(ns, dtype=dtype) + 0.1 * torch.randn(ns, ns, generator=g, dtype=dtype)).to(dev).requires_grad_()
    B = torch.randn(ns, nc, generator=g, dtype=dtype).to(dev).requires_grad_()
    x0 = torch.randn(nb, ns, generator=g, dtype=dtype).to(dev)
    lti = pp.module.LTI(A, B, torch.eye(ns, dtype=dtype, device=dev), torch.zeros(ns, nc, dtype=dtype, device=dev))
    return lti, Q, p, x0, (Q, p, A, B)


def run(lqr, x0, leaves, bwd, generic):
    if generic:
        K, k = lqr.lqr_backward(x0, 1)
        x, u, cost = lqr.lqr_forward(x0, K, k)
    else:
        x, u, cost = lqr(x0)
    if bwd:
        torch.autograd.grad(cost.sum() + x.sum(), leaves)


def timeit(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps * 1e-3


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("# device:", q.stdout.strip() or torch.cuda.get_device_name(dev))
    T = 100
    sizes = [1000, 10000] if "--quick" in sys.argv else [1000, 10000, 100000]
    print(f"{'dtype':6} {'ns,nc':6} {'B':>7} {'pass':8} {'cuda ms':>9} {'Mstep/s':>9} {'generic ms':>11} {'speedup':>8}")
    for dtype in (torch.float32, torch.float64):
        for ns, nc in ((4, 3), (12, 4)):
            for nb in sizes:
                lti, Q, p, x0, leaves = problem(nb, T, ns, nc, dtype, dev)
                lqr = pp.module.LQR(lti, Q, p, T)
                for bwd in (False, True):
                    tc = timeit(lambda: run(lqr, x0, leaves, bwd, False), 10)
                    tg = timeit(lambda: run(lqr, x0, leaves, bwd, True), 2) if nb <= 10000 else float("nan")
                    print(f"{str(dtype)[6:]:6} {ns},{nc:<4} {nb:>7} {'fwd+bwd' if bwd else 'fwd':8} {tc * 1e3:9.3f} "
                          f"{nb * T / tc / 1e6:9.2f} {tg * 1e3:11.2f} {tg / tc:8.1f}", flush=True)


if __name__ == "__main__":
    main()
