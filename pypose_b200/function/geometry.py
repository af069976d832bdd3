"""Projection / reprojection residual models and point-cloud functions (reference: pypose/function/geometry.py).

The camera-model functions the LM configs use (SURVEY.md §2 row 12), `svdtf`, which EPnP (SURVEY.md §8f.4, module/pnp.py)
needs, and `knn`, the brute-force nearest-neighbour search behind ICP (csrc/knn.cu, DESIGN.md §3.4).  The point-cloud
filters are not built.
"""
import ctypes
import math

import torch

from .. import _C
from ..basics import pm
from .checking import is_lietensor

torch.library.define("b200pose::knn", "(Tensor ref, Tensor nbr, int k, int ord, bool largest) -> (Tensor, Tensor)")

_ORD = {1: 1, 2: 2, math.inf: 0}


def _bstride(t):
    return 0 if t.shape[0] == 1 else t.shape[1] * t.shape[2]


@torch.library.impl("b200pose::knn", "CUDA")
def _knn_cuda(ref, nbr, k, ord, largest):
    """ref (B|1, N1, D), nbr (B|1, N2, D) contiguous, same dtype -> values (B, N1, k), int64 indices (B, N1, k)."""
    B, N1, N2, D = max(ref.shape[0], nbr.shape[0]), ref.shape[1], nbr.shape[1], ref.shape[2]
    vals = torch.empty(B, N1, k, dtype=ref.dtype, device=ref.device)
    idx = torch.empty(B, N1, k, dtype=torch.int64, device=ref.device)
    if B * N1 == 0:
        return vals, idx
    with torch.cuda.device(ref.device):
        q = _C.lib().b200_knn_workspace_bytes
        q.restype, q.argtypes = ctypes.c_longlong, [ctypes.c_longlong] * 6
        nws = int(q(B, N1, N2, D, k, ref.element_size()))
        ws = torch.empty(nws, dtype=torch.uint8, device=ref.device) if nws else None
        sym = f"b200_knn_{_C.suffix(ref.dtype)}"
        _C.check(_C.fn(sym)(ref.data_ptr(), _bstride(ref), nbr.data_ptr(), _bstride(nbr), vals.data_ptr(), idx.data_ptr(),
                            ws.data_ptr() if ws is not None else None, B, N1, N2, D, k, ord, int(largest),
                            _C.stream_ptr(ref.device)), sym)
    return vals, idx


@torch.library.register_fake("b200pose::knn")
def _knn_fake(ref, nbr, k, ord, largest):
    B, N1 = max(ref.shape[0], nbr.shape[0]), ref.shape[1]
    return ref.new_empty(B, N1, k), ref.new_empty(B, N1, k, dtype=torch.int64)


def _pc_batch(ref, nbr, B):
    """(..., N, D) -> (1 | prod(B), N, D) contiguous: an operand with one batch element is broadcast by stride 0."""
    def flat(t):
        lead = t.shape[:-2]
        if math.prod(lead) == 1:
            return t.reshape(1, *t.shape[-2:]).contiguous()
        return t.expand(*B, *t.shape[-2:]).reshape(math.prod(B), *t.shape[-2:]).contiguous()
    return flat(ref), flat(nbr)


def cart2homo(coordinates: torch.Tensor):
    """Append a homogeneous 1 (geometry.py:7-34)."""
    return torch.cat([coordinates, torch.ones_like(coordinates[..., :1])], dim=-1)


def homo2cart(coordinates: torch.Tensor):
    """Divide by the last coordinate, sign-preserving clamp away from 0 (geometry.py:37-57)."""
    last = coordinates[..., -1:]
    denom = pm(last) * last.abs().clamp_(min=torch.finfo(coordinates.dtype).tiny)
    return coordinates[..., :-1] / denom


def point2pixel(points, intrinsics, extrinsics=None):
    """Pinhole projection of (..., N, 3) points with (..., 3, 3) intrinsics (geometry.py:60-112)."""
    assert points.size(-1) == 3, "Points shape incorrect"
    assert intrinsics.size(-1) == intrinsics.size(-2) == 3, "Intrinsics shape incorrect."
    if extrinsics is None:
        torch.broadcast_shapes(points.shape[:-2], intrinsics.shape[:-2])
    else:
        assert is_lietensor(extrinsics) and extrinsics.shape[-1] == 7, "Type incorrect."
        torch.broadcast_shapes(points.shape[:-2], intrinsics.shape[:-2], extrinsics.shape[:-1])
        points = extrinsics.unsqueeze(-2) @ points
    return homo2cart(points @ intrinsics.mT)


def pixel2point(pixels, depth, intrinsics):
    """Back-projection of (..., N, 2) pixels with (..., N) depths through (..., 3, 3) pinhole intrinsics to (..., N, 3)
    camera-frame points: z = depth, x = (u - cx) z / fx, y = (v - cy) z / fy (geometry.py:115-168)."""
    assert pixels.size(-1) == 2, "Pixels shape incorrect"
    assert depth.size(-1) == pixels.size(-2), "Depth shape does not match pixels"
    assert intrinsics.size(-1) == intrinsics.size(-2) == 3, "Intrinsics shape incorrect."
    focal = torch.stack([intrinsics[..., 0, 0], intrinsics[..., 1, 1]], dim=-1)
    assert not torch.any(focal == 0), "fx / fy cannot contain zero"
    centre = intrinsics[..., :2, 2]
    xy = (pixels - centre.unsqueeze(-2)) * depth.unsqueeze(-1) / focal.unsqueeze(-2)
    return torch.cat([xy, depth.unsqueeze(-1)], dim=-1)


def reprojerr(points, pixels, intrinsics, extrinsics=None, reduction='none'):
    """Per-pixel reprojection error (geometry.py:171-225)."""
    torch.broadcast_shapes(points.shape[:-2], pixels.shape[:-2], intrinsics.shape[:-2])
    assert points.size(-1) == 3 and pixels.size(-1) == 2 and \
        intrinsics.size(-1) == intrinsics.size(-2) == 3, "Shape not compatible."
    assert reduction in {'norm', 'sum', 'none'}, "Reduction method can only be 'norm'|'sum'|'none'."
    err = point2pixel(points, intrinsics, extrinsics) - pixels
    if reduction == 'norm':
        return err.norm(dim=-1)
    if reduction == 'sum':
        return err.sum(dim=-1)
    return err


def knn(ref, nbr, k=1, ord=2, dim=-1, largest=False, sorted=True):
    """The k nearest (or, with `largest`, farthest) points of `nbr` (..., N2, D) for every point of `ref` (..., N1, D)
    under the `ord`-norm (1, 2 or inf) -> `torch.return_types.topk(values (..., N1, k), indices (..., N1, k))`, as the
    reference (geometry.py:228-313) computes with a (..., N1, N2, D) difference tensor and `topk`.

    Exact brute force on the GPU (csrc/knn.cu) without that tensor: D <= 16, k <= 32, batch dimensions broadcast.  The
    result is always sorted, and equal distances list the lower index first, so indices are deterministic; `sorted=False`
    is accepted and returns the same.  `values` is differentiable with respect to `ref` and `nbr`: when either requires
    grad the values are recomputed with torch ops from the selected neighbours (the selection itself has no gradient).

    Coordinates must be finite.  A candidate enters a list only if its distance compares strictly better, so a NaN
    distance never does: a query with NaN coordinates, or with fewer than k targets at a non-NaN distance, gets index -1
    and value inf (-inf with `largest`) in the slots left empty, where `torch.topk` would rank NaN as the largest value."""
    if not (isinstance(ref, torch.Tensor) and isinstance(nbr, torch.Tensor)):
        raise TypeError("knn: ref and nbr must be tensors")
    if not ref.is_cuda or not nbr.is_cuda:
        raise NotImplementedError(f"knn: expected CUDA tensors (no CPU path), got {ref.device} / {nbr.device}")
    if ref.device != nbr.device or ref.dtype != nbr.dtype:
        raise ValueError(f"knn: ref and nbr must share device and dtype, got {ref.device}/{ref.dtype} and {nbr.device}/{nbr.dtype}")
    _C.suffix(ref.dtype)
    if ref.dim() < 2 or nbr.dim() < 2:
        raise ValueError("knn: ref and nbr must have shape (..., N, D)")
    if dim not in (-1, ref.dim() - 1) or (dim == ref.dim() - 1 and ref.dim() != nbr.dim()):
        raise ValueError(f"knn: only the last dimension can hold the coordinates, got dim={dim}")
    if ord not in _ORD:
        raise ValueError(f"knn: ord must be 1, 2 or inf, got {ord}")
    D, N1, N2 = ref.shape[-1], ref.shape[-2], nbr.shape[-2]
    if nbr.shape[-1] != D:
        raise ValueError(f"knn: ref and nbr have different point dimensions {D} and {nbr.shape[-1]}")
    if not 1 <= D <= 16:
        raise ValueError(f"knn: point dimension must be 1..16, got {D}")
    if not isinstance(k, int) or k < 1 or k > 32:
        raise ValueError(f"knn: k must be an integer in 1..32, got {k}")
    if k > N2:
        raise ValueError(f"knn: k = {k} exceeds the number of neighbours N2 = {N2}")
    B = torch.broadcast_shapes(ref.shape[:-2], nbr.shape[:-2])
    if math.prod(B) == 0:
        vals = ref.new_empty(*B, N1, k)
        idx = torch.empty(*B, N1, k, dtype=torch.int64, device=ref.device)
    else:
        r, n = _pc_batch(ref.detach(), nbr.detach(), B)
        vals, idx = torch.ops.b200pose.knn(r, n, k, _ORD[ord], bool(largest))
        vals, idx = vals.view(*B, N1, k), idx.view(*B, N1, k)
    if torch.is_grad_enabled() and (ref.requires_grad or nbr.requires_grad):
        nb = nbr.expand(*B, N2, D)
        found = idx >= 0                  # see the docstring: -1 marks a slot no finite distance filled
        sel = torch.gather(nb, -2, idx.clamp(min=0).reshape(*B, N1 * k, 1).expand(*B, N1 * k, D)).view(*B, N1, k, D)
        diff = torch.where(found.unsqueeze(-1), ref.expand(*B, N1, D).unsqueeze(-2) - sel, 0)    # no NaN in the graph
        vals = torch.where(found, torch.linalg.vector_norm(diff, ord=ord, dim=-1), vals)
    return torch.return_types.topk((vals, idx))


def svdtf(source, target):
    """Rigid alignment of two associated point sets (..., N, 3) -> SE3 `T` with `T @ source ~ target`
    (geometry.py:315-358): rotation from the SVD of the cross-covariance of the centred sets.  Kept quirk: an improper
    solution (det = -1) is negated as a whole, as the reference does (:353-354), not by flipping one singular vector."""
    from ..lietensor import mat2SE3
    assert source.size(-2) == target.size(-2), "The number of points N has to be the same for both point clouds."
    cs, ct = source.mean(dim=-2, keepdim=True), target.mean(dim=-2, keepdim=True)
    cov = (target - ct).mT @ (source - cs)                       # (..., 3, 3): sum_n target_n source_n^T
    U, _, Vh = torch.linalg.svd(cov)
    R = U @ Vh
    improper = (torch.linalg.det(R) + 1).abs() < 1e-6
    R = torch.where(improper[..., None, None], -R, R)
    t = ct.mT - R @ cs.mT
    return mat2SE3(torch.cat([R, t], dim=-1), check=False)
