"""k-NN and ICP throughput on one GPU (csrc/knn.cu), with the reference formulation for comparison.

    python tools/bench_icp.py [--quick]

Prints one JSON line per measurement and the card name, power limit and max SM clock read in the same run.
* knn: pairs/s = B N1 N2 / kernel time (k = 1, ord 2, D = 3), fp32 and fp64, and the share of the issue bound of the
  FP32 (or FP64) pipe: the inner loop issues about 9 FP32 instructions per pair (3 FADD, FMUL, 2 FFMA, FSETP, 2 selects)
  in fp32 and 7 FP64 ones (3 DADD, DMUL, 2 DFMA, DSETP) in fp64, against 128 FP32 / 64 FP64 lanes per SM and clock at
  the card's max SM clock.
* reference: `torch.linalg.norm(ref[..., :, None, :] - nbr[..., None, :, :], dim=-1).topk(1, largest=False)`, as
  pypose/function/geometry.py:311-313 computes it, on the same GPU where it fits in memory.
* ICP: a fixed 30 iterations (ReduceToBason(30) with tol < 0 and a patience it cannot reach), device-decided loop; time
  per iteration and end to end (host call to result).
* ICP gradients (`--grad`, or `--grad-only`): the same runs with the source and target requiring grad and the loss
  sum W * T.matrix(): the forward with its trace, the backward, forward + backward, and the reference's formulation
  (oracle/icp_grad_oracle.py: knn through the difference tensor, torch.linalg.svd, autograd) where it fits in memory.
  The SM clock is sampled right after the timed runs.
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
from oracle import icp_grad_oracle as O  # noqa: E402

FP_INSTR = {torch.float32: (9, 128), torch.float64: (7, 64)}    # instructions per pair, lanes per SM and clock


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, plim, clk = [s.strip() for s in q.split(",")]
    return {"card": name, "power_limit_w": float(plim), "max_sm_clock_mhz": float(clk),
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def timed(fn, min_time=0.5, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    n, total = 0, 0.0
    while total < min_time:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1) / 1e3
        n += 1
    return total / n


def bench_knn(info, dt, B, N1, N2, quick):
    g = torch.Generator(device="cuda").manual_seed(0)
    r = torch.rand(B, N1, 3, device="cuda", dtype=dt, generator=g)
    n = torch.rand(B, N2, 3, device="cuda", dtype=dt, generator=g)
    t = timed(lambda: pp.knn(r, n), min_time=0.2 if quick else 1.0)
    pairs = B * N1 * N2 / t
    instr, lanes = FP_INSTR[dt]
    bound = info["sms"] * lanes * info["max_sm_clock_mhz"] * 1e6 / instr
    out = {"what": "knn", "dtype": str(dt).split(".")[1], "B": B, "N1": N1, "N2": N2, "k": 1, "time_ms": t * 1e3,
           "pairs_per_s": pairs, "share_of_issue_bound": pairs / bound}
    try:
        def reference():
            return torch.linalg.norm(r.unsqueeze(-2) - n.unsqueeze(-3), dim=-1).topk(1, dim=-1, largest=False)
        ref = reference()
        mine = pp.knn(r, n)
        out["reference_time_ms"] = timed(reference, min_time=0.2 if quick else 1.0, warmup=1) * 1e3
        out["reference_values_match"] = bool(torch.allclose(ref.values, mine.values, rtol=1e-5, atol=1e-6))
        del ref
    except torch.OutOfMemoryError:
        out["reference_time_ms"] = None                  # the difference tensor does not fit
    torch.cuda.empty_cache()
    return out


def bench_icp(dt, B, N, iters=30):
    g = torch.Generator(device="cuda").manual_seed(1)
    xy = torch.rand(B, N, 2, device="cuda", dtype=torch.float64, generator=g) * 10
    tgt = torch.cat([xy, torch.sin(xy[..., :1]) + torch.cos(0.7 * xy[..., 1:])], -1)
    tf = pp.se3(0.02 * torch.randn(B, 6, device="cuda", dtype=torch.float64, generator=g)).Exp()
    src = tf.Inv().unsqueeze(-2).Act(tgt).to(dt)
    tgt = tgt.to(dt)
    stepper = pp.utils.ReduceToBason(iters, patience=10 ** 9, tol=-1.0)
    icp = pp.module.ICP(stepper=stepper)
    icp(src, tgt)
    torch.cuda.synchronize()
    runs = []
    for _ in range(5):
        t0 = time.perf_counter()
        icp(src, tgt)
        torch.cuda.synchronize()
        runs.append(time.perf_counter() - t0)
    assert stepper.steps == iters
    t = sorted(runs)[len(runs) // 2]
    return {"what": "icp", "dtype": str(dt).split(".")[1], "B": B, "N": N, "iterations": iters, "end_to_end_ms": t * 1e3,
            "per_iteration_us": t / iters * 1e6, "pairs_per_s": B * N * N * iters / t}


def sm_clock():
    return float(subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i",
                                 str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip())


def median_time(fn, n=5):
    runs = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        runs.append(time.perf_counter() - t0)
    return sorted(runs)[len(runs) // 2]


def bench_icp_grad(dt, B, N, iters=30):
    g = torch.Generator(device="cuda").manual_seed(1)
    xy = torch.rand(B, N, 2, device="cuda", dtype=torch.float64, generator=g) * 10
    tgt = torch.cat([xy, torch.sin(xy[..., :1]) + torch.cos(0.7 * xy[..., 1:])], -1)
    tf = pp.se3(0.02 * torch.randn(B, 6, device="cuda", dtype=torch.float64, generator=g)).Exp()
    src = tf.Inv().unsqueeze(-2).Act(tgt).to(dt).requires_grad_()
    tgt = tgt.to(dt).requires_grad_()
    W = torch.randn(B, 4, 4, device="cuda", dtype=dt, generator=None)
    stepper = pp.utils.ReduceToBason(iters, patience=10 ** 9, tol=-1.0)
    icp = pp.module.ICP(stepper=stepper)
    box = {}

    def fwd():
        box["L"] = (icp(src, tgt).matrix() * W).sum()

    def bwd():
        torch.autograd.grad(box["L"], [src, tgt])

    def both():
        fwd()
        bwd()
    both()
    assert stepper.steps == iters
    t_fwd = median_time(fwd)
    t_bwd_runs = []
    for _ in range(5):
        fwd()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        bwd()
        torch.cuda.synchronize()
        t_bwd_runs.append(time.perf_counter() - t0)
    t_bwd = sorted(t_bwd_runs)[2]
    t_both = median_time(both)
    clk = sm_clock()
    out = {"what": "icp_grad", "dtype": str(dt).split(".")[1], "B": B, "N": N, "iterations": iters,
           "forward_with_trace_ms": t_fwd * 1e3, "backward_ms": t_bwd * 1e3, "forward_backward_ms": t_both * 1e3,
           "sm_clock_mhz_after": clk}
    box.clear()
    torch.cuda.empty_cache()
    try:
        def reference():
            T, _ = O.icp(src, tgt, iters, None, 2, "project")
            torch.autograd.grad((O.Matrix.apply(T) * W).sum(), [src, tgt])
        reference()
        out["reference_forward_backward_ms"] = median_time(reference, 3) * 1e3
    except torch.OutOfMemoryError:
        out["reference_forward_backward_ms"] = None        # the difference tensor does not fit
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="shorter timing windows")
    ap.add_argument("--grad", action="store_true", help="also the ICP gradient rows")
    ap.add_argument("--grad-only", action="store_true", help="only the ICP gradient rows")
    a = ap.parse_args()
    info = card()
    print(json.dumps(info), flush=True)
    if a.grad or a.grad_only:
        for dt in (torch.float32, torch.float64):
            for B, N in ((1, 100000), (64, 4096)):
                print(json.dumps({**bench_icp_grad(dt, B, N), "card": info["card"], "power_limit_w": info["power_limit_w"]}),
                      flush=True)
        if a.grad_only:
            return
    for dt in (torch.float32, torch.float64):
        for B, N1, N2 in ((1, 100000, 100000), (64, 4096, 4096), (1, 20000, 200000)):
            print(json.dumps({**bench_knn(info, dt, B, N1, N2, a.quick), "card": info["card"],
                              "power_limit_w": info["power_limit_w"]}), flush=True)
    for dt in (torch.float32, torch.float64):
        for B, N in ((1, 100000), (64, 4096)):
            print(json.dumps({**bench_icp(dt, B, N), "card": info["card"], "power_limit_w": info["power_limit_w"]}), flush=True)


if __name__ == "__main__":
    main()
