"""Point-cloud filter timings on one GPU (csrc/voxel.cu, the radius mask of csrc/knn.cu), with the reference
formulations for comparison.

    python tools/bench_pcfilter.py [--quick]

Prints the card name, power limit and max SM clock read in the same run, then one JSON line per measurement.  Every
time is end to end per call (host clock around the call and a device synchronise), host reads included.
* voxel_filter (centroids, fp32) at N = 1.2e5, 1e6, 1e7, D = 3 and 4, uniform points in a cube with a voxel size that
  gives about N / 10 voxels; `reference`: minimum, integer coordinates, `torch.unique(dim=-2)` and `index_add_` as
  pypose/function/geometry.py:579-602 computes them, on the same GPU.  Also the whole cloud in one voxel (one thread
  sums it) at 1e6 and 1e7 points.
* voxel_filter(random=True) against the reference's per-voxel loop of `randint(count.item())` (one host sync per voxel)
  at M ~ 1000 voxels only.
* nbr_filter at N = 1.2e5: a uniform cloud where almost no point reaches `nbr` (every CTA scans every tile) and a
  clustered one (CTAs stop early); pairs/s = N^2 / time.  The reference formulation ((N, N, 3) difference tensor) is
  timed at N = 2e4, where it fits.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, plim, clk = [s.strip() for s in q.split(",")]
    return {"card": name, "power_limit_w": float(plim), "max_sm_clock_mhz": float(clk),
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def timed(fn, min_time=0.5, warmup=2, max_runs=200):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    runs = []
    while sum(runs) < min_time and len(runs) < max_runs:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        runs.append(time.perf_counter() - t0)
    return sorted(runs)[len(runs) // 2]


def ref_voxel(points, voxel):
    vdim, D = len(voxel), points.shape[1]
    minp = torch.min(points[..., :vdim], dim=-2).values
    idx = ((points[..., :vdim] - minp) / torch.tensor(voxel, device=points.device)).to(torch.int64)
    uniq, inv = torch.unique(idx, dim=-2, return_inverse=True)
    vox = torch.zeros(len(uniq), D, dtype=points.dtype, device=points.device)
    cnt = torch.zeros(len(uniq), dtype=points.dtype, device=points.device)
    vox.index_add_(0, inv, points)
    cnt.index_add_(0, inv, torch.ones_like(inv, dtype=points.dtype))
    return vox / cnt.view(-1, 1)


def ref_voxel_random(points, voxel):
    vdim = len(voxel)
    minp = torch.min(points[..., :vdim], dim=-2).values
    idx = ((points[..., :vdim] - minp) / torch.tensor(voxel, device=points.device)).to(torch.int64)
    _, inv, counts = torch.unique(idx, dim=-2, return_inverse=True, return_counts=True)
    sp = points[torch.argsort(inv)]
    r = torch.cat([torch.randint(0, c.item(), (1,), device=points.device) for c in counts])
    return sp[r + torch.cumsum(counts, 0) - counts]


def ref_nbr(points, nbr, radius):
    d = torch.linalg.norm(points.unsqueeze(-2) - points.unsqueeze(-3), dim=-1)
    return points[(d <= radius).sum(-1) - 1 >= nbr]


def bench_voxel(N, D, quick, one_voxel=False):
    g = torch.Generator(device="cuda").manual_seed(N + D)
    L = 10.0
    pts = torch.rand(N, D, device="cuda", generator=g) * L
    s = L / (N / 10) ** (1 / 3)
    vox = [100 * L] * 3 if one_voxel else [s] * 3
    out = pp.voxel_filter(pts, vox)
    t = timed(lambda: pp.voxel_filter(pts, vox), min_time=0.2 if quick else 1.0)
    res = {"what": "voxel_filter", "dtype": "float32", "N": N, "D": D, "voxels": out.shape[0], "time_ms": t * 1e3,
           "points_per_s": N / t}
    if not one_voxel:
        try:
            r = ref_voxel(pts, vox)
            res["reference_max_abs_diff"] = float((r - out).abs().max())
            res["reference_time_ms"] = timed(lambda: ref_voxel(pts, vox), min_time=0.2 if quick else 1.0, warmup=1) * 1e3
            del r
        except torch.OutOfMemoryError:
            res["reference_time_ms"] = None
    torch.cuda.empty_cache()
    return res


def bench_voxel_random(quick):
    g = torch.Generator(device="cuda").manual_seed(3)
    pts = torch.rand(20000, 3, device="cuda", generator=g) * 10
    vox = [1.0, 1.0, 1.0]                                  # 1000 voxels
    M = pp.voxel_filter(pts, vox, random=True).shape[0]
    t = timed(lambda: pp.voxel_filter(pts, vox, random=True), min_time=0.2 if quick else 1.0)
    tr = timed(lambda: ref_voxel_random(pts, vox), min_time=0.2 if quick else 1.0, warmup=1, max_runs=10)
    return {"what": "voxel_filter_random", "dtype": "float32", "N": 20000, "voxels": M, "time_ms": t * 1e3,
            "reference_time_ms": tr * 1e3}


def bench_nbr(N, clustered, quick, with_reference=False):
    g = torch.Generator(device="cuda").manual_seed(N + clustered)
    if clustered:                                          # 100 dense clusters in random index order, 1 % outliers
        c = torch.rand(100, 3, device="cuda", generator=g) * 100
        n_in = N - N // 100
        pts = c.repeat_interleave(n_in // 100, 0) + 0.3 * torch.randn(n_in, 3, device="cuda", generator=g)
        pts = torch.cat([pts[torch.randperm(n_in, device="cuda", generator=g)],
                         torch.rand(N - n_in, 3, device="cuda", generator=g) * 100])
        nbr, radius = 16, 1.0
    else:                                                  # about 4 neighbours per point: almost every point fails
        pts = torch.rand(N, 3, device="cuda", generator=g) * 100
        nbr, radius = 16, 100 * (3 * 4 / (4 * 3.14159 * N)) ** (1 / 3)
    kept = int(pp.nbr_filter(pts, nbr, radius, return_mask=True)[1].sum())
    t = timed(lambda: pp.nbr_filter(pts, nbr, radius), min_time=0.2 if quick else 1.0)
    res = {"what": "nbr_filter", "dtype": "float32", "N": N, "cloud": "clustered" if clustered else "uniform",
           "nbr": nbr, "radius": radius, "kept": kept, "time_ms": t * 1e3, "pairs_per_s": N * N / t}
    if with_reference:
        try:
            r = ref_nbr(pts, nbr, radius)
            res["reference_kept"] = r.shape[0]
            res["reference_time_ms"] = timed(lambda: ref_nbr(pts, nbr, radius), min_time=0.2 if quick else 1.0,
                                             warmup=1) * 1e3
            del r
        except torch.OutOfMemoryError:
            res["reference_time_ms"] = None
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="shorter timing windows")
    a = ap.parse_args()
    info = card()
    print(json.dumps(info), flush=True)
    tag = {"card": info["card"], "power_limit_w": info["power_limit_w"]}
    for N in (120000, 1000000, 10000000):
        for D in (3, 4):
            print(json.dumps({**bench_voxel(N, D, a.quick), **tag}), flush=True)
    for N in (1000000, 10000000):
        print(json.dumps({**bench_voxel(N, 3, a.quick, one_voxel=True), "one_voxel": True, **tag}), flush=True)
    print(json.dumps({**bench_voxel_random(a.quick), **tag}), flush=True)
    for clustered in (False, True):
        print(json.dumps({**bench_nbr(120000, clustered, a.quick), **tag}), flush=True)
        print(json.dumps({**bench_nbr(20000, clustered, a.quick, with_reference=True), **tag}), flush=True)


if __name__ == "__main__":
    main()
