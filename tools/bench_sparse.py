"""Time pp.bsr_bsc_matmul (forward, and forward + backward through the values) on three block-sparse workloads, against
torch's CUDA CSR × CSR product of the element-wise expanded matrices and, where the dense result fits, dense
torch.matmul.  Prints the card and its power limit, then one JSON line per workload.

    python tools/bench_sparse.py [--reps 5] [--dtype float32|float64] [--scale 1.0]

Workloads (scale multiplies the block counts):
  random    A @ A.mT, a 1e5 × 1e5 grid of 6 × 6 blocks with 8 random blocks per row
  banded    A @ A.mT, a pose-graph-like 1e5-block matrix: the diagonal, the next block and one random loop closure per row
  reproj    J @ J.mT, a reprojection-shaped J: 2 × 6 blocks, 1000 cameras with 64 observations each, one camera per row
The maximum difference is |C x - C_ref x| / |C_ref x| (max norm) for a random dense x, at the timed sizes.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pypose_b200 as pp  # noqa: E402
from pypose_b200.sparse.ops import _BsrBscValues  # noqa: E402

warnings.filterwarnings("ignore", message=".*Sparse.*")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


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


def bsr_from_cols(cols, ncols, block, dtype, dev, g):
    """BSR with block row i holding the (sorted, unique) block columns cols[i] (a (rows, k) tensor, -1 = none)."""
    rows = cols.shape[0]
    cols, _ = torch.sort(cols, 1)
    keep = cols >= 0
    keep[:, 1:] &= cols[:, 1:] != cols[:, :-1]
    crow = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(keep.sum(1), 0)])
    col = cols[keep]
    val = torch.randn(col.numel(), *block, dtype=dtype, device=dev, generator=g)
    return torch.sparse_bsr_tensor(crow, col, val, size=(rows * block[0], ncols * block[1]))


def workloads(scale, dtype, dev, g):
    n = int(1e5 * scale)
    yield "random", bsr_from_cols(torch.randint(0, n, (n, 8), device=dev, generator=g), n, (6, 6), dtype, dev, g)
    i = torch.arange(n, device=dev)
    cols = torch.stack([i, torch.where(i + 1 < n, i + 1, -1), torch.randint(0, n, (n,), device=dev, generator=g)], 1)
    yield "banded", bsr_from_cols(cols, n, (6, 6), dtype, dev, g)
    ncam, per = int(1000 * scale), 64
    cam = torch.arange(ncam, device=dev).repeat_interleave(per)[torch.randperm(ncam * per, device=dev, generator=g)]
    yield "reproj", bsr_from_cols(cam[:, None], ncam, (2, 6), dtype, dev, g)


def apply_bsr(C, x):
    """C x for a BSR C and a dense (p, r) x, in torch ops (no vendor BSR kernel)."""
    dm, dp = C.values().shape[1:]
    crow = C.crow_indices()
    rows = torch.repeat_interleave(torch.arange(crow.numel() - 1, device=x.device), crow.diff())
    xb = x.view(-1, dp, x.shape[1])[C.col_indices()]
    y = torch.zeros(crow.numel() - 1, dm, x.shape[1], dtype=x.dtype, device=x.device)
    y.index_add_(0, rows, torch.bmm(C.values(), xb))
    return y.view(-1, x.shape[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dtype", default="float64", choices=["float32", "float64"])
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--dense-max-gb", type=float, default=8.0)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    dtype = getattr(torch, a.dtype)
    g = torch.Generator(device=dev).manual_seed(0)
    print("card:", card(), flush=True)
    for name, A in workloads(a.scale, dtype, dev, g):
        B = A.mT
        C = pp.bsr_bsc_matmul(A, B)
        rec = {"what": name, "dtype": a.dtype, "shape": list(A.shape), "block": list(A.values().shape[1:]),
               "nnz_blocks_A": A.values().shape[0], "nnz_blocks_C": C.values().shape[0]}
        rec["fwd_ms"] = round(1e3 * timed(lambda: pp.bsr_bsc_matmul(A, B), a.reps), 3)
        v = A.values().detach().clone().requires_grad_()
        crow, col = A.crow_indices(), A.col_indices()

        sm, sn = A.shape[0] // A.values().shape[1], A.shape[1] // A.values().shape[2]

        def fwd_bwd():          # the values-level Function: torch's sparse autograd would form dense (m, m) tensors
            c = _BsrBscValues.apply(v, None, crow, col, crow, col, sm, sn, sm)[0]
            (gv,) = torch.autograd.grad(c.sum(), v)
            return gv
        rec["fwd_bwd_ms"] = round(1e3 * timed(fwd_bwd, a.reps), 3)
        x = torch.randn(C.shape[1], 4, dtype=dtype, device=dev, generator=g)
        y = apply_bsr(C, x)
        try:
            Ae = A.to_sparse_coo().coalesce().to_sparse_csr()            # element-wise expanded
            Be = A.mT.to_sparse_coo().coalesce().to_sparse_csr()
            rec["torch_csr_ms"] = round(1e3 * timed(lambda: Ae @ Be, a.reps), 3)
            yt = (Ae @ Be) @ x
            rec["max_rel_diff_vs_torch_csr"] = float((y - yt).abs().max() / yt.abs().max())
            del Ae, Be, yt
        except (RuntimeError, torch.OutOfMemoryError) as e:
            rec["torch_csr_ms"] = f"failed: {str(e).splitlines()[0][:120]}"
        if C.shape[0] * C.shape[1] * A.values().element_size() * 3 <= a.dense_max_gb * 2**30:
            Ad = A.to_dense()
            rec["dense_matmul_ms"] = round(1e3 * timed(lambda: Ad @ Ad.mT, a.reps), 3)
            yd = (Ad @ Ad.mT) @ x
            rec["max_rel_diff_vs_dense"] = float((y - yd).abs().max() / yd.abs().max())
            del Ad
        else:
            rec["dense_matmul_ms"] = "does not fit"
        print(json.dumps(rec), flush=True)
        del A, B, C
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
