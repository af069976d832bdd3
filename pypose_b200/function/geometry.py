"""Projection / reprojection residual models and point-cloud functions (reference: pypose/function/geometry.py).

The camera-model functions the LM configs use (SURVEY.md §2 row 12), `svdtf`, which EPnP (SURVEY.md §8f.4, module/pnp.py)
needs, `svdstf` (Umeyama Sim3 alignment), `knn`, the brute-force nearest-neighbour search behind ICP (csrc/knn.cu,
DESIGN.md §3.4), and the point-cloud filters (DESIGN.md §3.5): `nbr_filter` and `knn_filter` on a radius count in
csrc/knn.cu, `voxel_filter` on the sort-and-reduce pipeline of csrc/voxel.cu, and `random_filter`.
"""
import ctypes
import math

import numpy as np
import torch

from .. import _C
from ..basics import pm
from .checking import is_lietensor

torch.library.define("b200pose::knn", "(Tensor ref, Tensor nbr, int k, int ord, bool largest) -> (Tensor, Tensor)")
torch.library.define("b200pose::radius_mask", "(Tensor pts, float thr, int ord, int need) -> Tensor")

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
    and value inf (-inf with `largest`) in the slots left empty, where `torch.topk` would rank NaN as the largest value.
    A NaN in any coordinate makes the distance NaN, for every `ord`."""
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


def svdstf(source, target, with_scale=True):
    """Similarity alignment of two associated point sets (..., N, 3) -> Sim3 `T` with `T @ source ~ target`, by
    Umeyama's method as the reference computes it (geometry.py:361-432): H = t^T s / N of the centred sets, M = diag(1, 1,
    sign det(U Vh)), scale = sum(diag(M) sigma) / var(s) (1 without `with_scale`), R = U M Vh, t = c_t - scale R c_s.

    Torch ops on any device.  Difference from the reference: M is built on the inputs' device (the reference builds it
    on the CPU, so CUDA inputs would mix devices in `U @ M @ V`)."""
    from ..lietensor import mat2Sim3
    assert source.size(-2) == target.size(-2), "The number of points N has to be the same for both point clouds."
    assert source.size(-1) == 3 and target.size(-1) == 3, "The point dimension has to be 3."
    N, m = source.shape[-2:]
    cs, ct = source.mean(dim=-2, keepdim=True), target.mean(dim=-2, keepdim=True)
    s_, t_ = source - cs, target - ct
    H = t_.mT @ s_ / N
    U, D, V = torch.linalg.svd(H)
    M = torch.eye(m, dtype=U.dtype, device=U.device).expand_as(U).clone()
    M[..., -1, -1] = torch.sign(torch.det(U @ V))
    if with_scale:
        var = (s_.norm(dim=-1) ** 2).mean(dim=-1, keepdim=True)
        scale = torch.sum(torch.diagonal(M, dim1=-1, dim2=-2) * D, keepdim=True, dim=-1) / var
    else:
        scale = torch.ones_like(D[..., 0:1])
    scale = scale.unsqueeze(-1)
    R = U @ M @ V
    t = ct.mT - scale * R @ cs.mT
    return mat2Sim3(torch.cat((scale * R, t), dim=-1), check=True)


def _np_dtype(dtype):
    return np.float32 if dtype == torch.float32 else np.float64


def _sq_threshold(radius, dtype):
    """The ord-2 radius test `sqrt(d2) <= r` (r = `radius` rounded to `dtype`, sqrt correctly rounded) as `d2 <= t`: the
    largest t of `dtype` with sqrt(t) <= r, found by stepping from r * r with nextafter (sqrt is monotone, so both tests
    decide alike).  -1 when no distance passes (r < 0 or NaN)."""
    ft = _np_dtype(dtype)
    r = ft(radius)
    if not r >= 0:
        return -1.0
    if np.isinf(r):
        return math.inf
    up, down = ft(np.inf), ft(-np.inf)
    with np.errstate(over="ignore"):
        t = ft(r * r)
        while np.sqrt(t) > r:
            t = np.nextafter(t, down)
        while True:
            nt = np.nextafter(t, up)
            if not np.isfinite(nt) or np.sqrt(nt) > r:
                break
            t = nt
    return float(t)


@torch.library.impl("b200pose::radius_mask", "CUDA")
def _radius_mask_cuda(pts, thr, ord, need):
    """pts (N, D) contiguous -> bool (N,): count of points within the threshold, itself included, >= need."""
    N, D = pts.shape
    mask = torch.empty(N, dtype=torch.bool, device=pts.device)
    if N == 0:
        return mask
    with torch.cuda.device(pts.device):
        sym = f"b200_radius_mask_{_C.suffix(pts.dtype)}"
        _C.check(_C.fn(sym)(pts.data_ptr(), N, D, float(thr), ord, need, mask.data_ptr(), _C.stream_ptr(pts.device)), sym)
    return mask


@torch.library.register_fake("b200pose::radius_mask")
def _radius_mask_fake(pts, thr, ord, need):
    return pts.new_empty(pts.shape[0], dtype=torch.bool)


def _check_cuda(name, points):
    if not points.is_cuda:
        raise NotImplementedError(f"{name}: expected a CUDA tensor (no CPU path), got {points.device}")
    _C.suffix(points.dtype)


def _pdim(name, points, pdim):
    D = points.shape[-1]
    pdim = D if pdim is None else pdim
    if not isinstance(pdim, int) or not 1 <= pdim <= D:
        raise ValueError(f"{name}: pdim must be an integer in 1..{D} (the last dimension of points), got {pdim}")
    if pdim > 16:
        raise ValueError(f"{name}: at most 16 coordinates take part in the distances, got pdim = {pdim}")
    return pdim


def _radius_mask(points, pdim, radius, ord, nbr):
    """Keep-mask of the points with at least `nbr` others within `radius` (the shared test of nbr_filter and knn_filter)."""
    radius = float(radius)
    thr = _sq_threshold(radius, points.dtype) if ord == 2 else float(_np_dtype(points.dtype)(radius))
    pts = points[:, :pdim].contiguous()
    return torch.ops.b200pose.radius_mask(pts, thr, _ORD[ord], int(nbr) + 1)


def nbr_filter(points, nbr, radius, pdim=None, ord=2, return_mask=False):
    """Radius outlier removal (geometry.py:436-493): keep the points of `points` (N, D) that have at least `nbr`
    neighbours, themselves excluded, whose `ord`-norm distance (1, 2 or inf) over the first `pdim` coordinates is
    <= `radius`.  Returns `points[mask]` (all D columns), and the bool `mask` (N,) with `return_mask`.

    A brute-force count on the GPU (csrc/knn.cu, DESIGN.md §3.5) without the reference's (N, N, pdim) difference
    tensor: fp32 / fp64 CUDA tensors, pdim <= 16.  `radius` is rounded to the points' dtype, as the reference's
    comparison does; for ord 2 the test is `sqrt(d2) <= radius` with a correctly rounded root, evaluated as `d2 <= t`
    with the largest such t.  Squared distances are summed with FMAs, so a point whose distance lies within a few units
    in the last place of `radius` may be decided differently from the reference.  Coordinates must be finite."""
    if not isinstance(points, torch.Tensor) or points.dim() != 2:
        raise ValueError("nbr_filter: points must be a tensor of shape (N, D)")
    pdim = _pdim("nbr_filter", points, pdim)
    if ord not in _ORD:
        raise ValueError(f"nbr_filter: ord must be 1, 2 or inf, got {ord}")
    _check_cuda("nbr_filter", points)
    mask = _radius_mask(points, pdim, radius, ord, nbr)
    return (points[mask], mask) if return_mask else points[mask]


def random_filter(points, num):
    """`num` points (..., num, D) drawn without replacement from `points` (..., N, D) (geometry.py:496-527).  The same
    indices apply to every batch element, as in the reference; the permutation is drawn on the points' device (the
    reference draws it on the CPU), so results differ from the reference's under the same seed.  Torch ops on any
    device."""
    if not isinstance(points, torch.Tensor) or points.dim() < 2 or points.shape[-1] < 1:
        raise ValueError("random_filter: points must be a tensor of shape (..., N, D)")
    N = points.shape[-2]
    if not isinstance(num, int) or not 0 <= num <= N:
        raise ValueError(f"random_filter: num must be an integer in 0..{N} (the number of points), got {num}")
    idx = torch.randperm(N, device=points.device)[:num]
    return points[..., idx, :]


def _voxel_plan(lo, hi):
    """Key layout of integer voxel coordinates in [lo_d, hi_d] per dimension: each dimension takes
    bit_length(hi_d - lo_d) bits and the dimensions are packed in order, the first most significant, into as few keys of
    at most 64 bits as hold them.  -> [(group, shift)] per dimension and the bit count of each group; comparing the
    group keys in order compares the coordinates lexicographically."""
    widths = [int(h - l).bit_length() for l, h in zip(lo, hi)]
    groups, bits = [], [0]
    for w in widths:
        if bits[-1] + w > 64:
            bits.append(0)
        groups.append(len(bits) - 1)
        bits[-1] += w
    shifts = []
    for d, g in enumerate(groups):
        shifts.append(sum(widths[e] for e in range(d + 1, len(widths)) if groups[e] == g))
    return list(zip(groups, shifts)), bits


def _voxel_ranges(mn, mx, v, dtype):
    """Per dimension, the integer range [lo, hi] of trunc((p - min) / v) over the points, from the extent computed with
    the same float subtract and divide.  Raises when an extent reaches 2^62 voxels."""
    ft = _np_dtype(dtype)
    lo, hi = [], []
    with np.errstate(all="ignore"):
        for a, b, s in zip(mn, mx, v):
            q = ft(ft(b) - ft(a)) / ft(s)
            if not np.isfinite(q) or abs(q) >= 2.0 ** 62:
                raise ValueError(f"voxel_filter: the cloud spans {abs(q)} voxels of size {s} in one dimension; "
                                 "coordinates must be finite and the extent below 2^62 voxels")
            c = int(q)
            lo.append(min(c, 0))
            hi.append(max(c, 0))
    return lo, hi


def _voxel_sort(points, voxel):
    """points (N, D) contiguous CUDA, N > 0 -> (workspace, voxel id of every point (N,) int64, number of voxels M)."""
    N, D = points.shape
    vdim = len(voxel)
    ft = _np_dtype(points.dtype)
    v = torch.tensor(voxel).to(points.dtype)                   # the default dtype first, as the reference does
    mn, mx = torch.aminmax(points[:, :vdim], dim=0)
    mm = torch.stack([mn, mx]).cpu().numpy()                   # the first host read
    vv = v.numpy()
    lo, hi = _voxel_ranges(mm[0], mm[1], vv, points.dtype)
    layout, bits = _voxel_plan(lo, hi)
    bounds = np.ascontiguousarray(np.stack([mm[0].astype(ft), vv.astype(ft)], 1).astype(np.float64).ravel())
    plan = np.array([x for d in range(vdim) for x in (lo[d], *layout[d])] + bits, dtype=np.int64)
    dev = points.device
    with torch.cuda.device(dev):
        q = _C.lib().b200_voxel_workspace_bytes
        q.restype, q.argtypes = ctypes.c_longlong, [ctypes.c_longlong]
        ws = torch.empty(int(q(N)), dtype=torch.uint8, device=dev)
        vid = torch.empty(N, dtype=torch.int64, device=dev)
        M = torch.empty(1, dtype=torch.int64, device=dev)
        sym = f"b200_voxel_sort_{_C.suffix(points.dtype)}"
        _C.check(_C.fn(sym)(points.data_ptr(), N, D, vdim, bounds.ctypes.data, plan.ctypes.data, len(bits), ws.data_ptr(),
                            vid.data_ptr(), M.data_ptr(), _C.stream_ptr(dev)), sym)
    return ws, vid, int(M.item())                              # the second host read


def _voxel_reduce(points, ws, M, u=None):
    """Centroids (M, D) and member counts (M,), or with uniforms `u` (M,) fp64 the picked rows (M,) int64."""
    N, D = points.shape
    dev = points.device
    out = cnt = sel = None
    if u is None:
        out = torch.empty(M, D, dtype=points.dtype, device=dev)
        cnt = torch.empty(M, dtype=points.dtype, device=dev)
    else:
        sel = torch.empty(M, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        sym = f"b200_voxel_reduce_{_C.suffix(points.dtype)}"
        ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        _C.check(_C.fn(sym)(points.data_ptr(), N, D, ws.data_ptr(), M, ptr(u), ptr(out), ptr(cnt), ptr(sel),
                            _C.stream_ptr(dev)), sym)
    return (out, cnt) if u is None else sel


class _VoxelCentroid(torch.autograd.Function):
    """Centroid mode of voxel_filter: the kernel's values forward; backward gives every point grad_out[its voxel] / count
    (the count as the forward divided by it)."""

    @staticmethod
    def forward(ctx, points, voxel):
        pts = points.detach().contiguous()
        ws, vid, M = _voxel_sort(pts, voxel)
        out, cnt = _voxel_reduce(pts, ws, M)
        ctx.save_for_backward(vid, cnt)
        return out

    @staticmethod
    def backward(ctx, grad):
        vid, cnt = ctx.saved_tensors
        return (grad / cnt.unsqueeze(-1))[vid], None


def voxel_filter(points, voxel, random=False):
    """One point per occupied voxel of `points` (N, D) -> (M, D) (geometry.py:530-602): the centroid of the voxel's
    points, or with `random` one of them chosen uniformly.  `voxel` holds the sizes of the first vdim = len(voxel) <= D
    coordinates; the voxel of a point is trunc((p - min) / voxel) per dimension, min over the cloud, with sizes passed
    through `torch.tensor(voxel)` (float32 by default) first and negative sizes allowed, as in the reference.  Voxels come
    in lexicographic order of their integer coordinates (the order of `torch.unique(dim=-2)`).

    On the GPU (csrc/voxel.cu, DESIGN.md §3.5): fp32 / fp64 CUDA tensors, vdim <= 16, two host reads per call (the
    coordinate ranges and the voxel count).  Centroids sum each voxel's points in increasing index order in the points'
    dtype, as the reference's `index_add_` on the CPU does, so they are deterministic and equal the reference run on the
    CPU bit for bit; a voxel holding most of the cloud is summed by one thread.  They are differentiable with respect to
    `points`.  `random` draws one uniform per voxel from torch's generator on the device and takes the member
    min(floor(u count), count - 1) in index order, with no per-voxel host sync; the result is always (M, D), where the
    reference squeezes a single voxel to (D,).  Coordinates must be finite, and every extent must stay below 2^62
    voxels (ValueError)."""
    if not isinstance(points, torch.Tensor) or points.dim() != 2:
        raise ValueError("voxel_filter: points must be a tensor of shape (N, D)")
    voxel = [float(s) for s in voxel]
    D, vdim = points.shape[-1], len(voxel)
    if not 1 <= vdim <= min(D, 16):
        raise ValueError(f"voxel_filter: len(voxel) must be in 1..min(16, D) with D = {D}, got {vdim}")
    if any(s == 0 for s in voxel):
        raise ValueError(f"voxel_filter: voxel sizes must be nonzero, got {voxel}")
    _check_cuda("voxel_filter", points)
    if points.shape[0] == 0:
        return points.new_empty(0, D)
    if not random:
        return _VoxelCentroid.apply(points, voxel)
    pts = points.detach().contiguous()
    ws, _, M = _voxel_sort(pts, voxel)
    u = torch.rand(M, dtype=torch.float64, device=points.device)
    return points[_voxel_reduce(pts, ws, M, u)]


def knn_filter(points, k, pdim=None, radius=None, ord=2):
    """Every point replaced by the mean, over all D columns, of itself and its k nearest neighbours in the first `pdim`
    coordinates under the `ord`-norm (geometry.py:605-664).  Without `radius`, batched: (..., N, D) -> (..., N, D).
    With `radius`, `points` is (N, D) and the points with fewer than k neighbours within `radius` (the test of
    `nbr_filter` with nbr = k) are removed first -> (M, D).

    The k + 1 neighbours come from `knn` (csrc/knn.cu; equal distances list the lower index first), the radius test from
    the kernel of `nbr_filter`: fp32 / fp64 CUDA tensors, k + 1 <= min(32, N), pdim <= 16.  Difference from the
    reference with `radius`: the neighbours of a kept point are searched in, and gathered from, the full cloud.  The
    reference gathers from the kept rows with indices into the full cloud, which agrees only when every selected index
    is below the number of kept rows and those rows are the cloud's first ones (as in its docstring example); otherwise
    it reads other rows or raises.  Coordinates must be finite."""
    if not isinstance(points, torch.Tensor) or points.dim() < 2 or (radius is not None and points.dim() != 2):
        raise ValueError("knn_filter: points must be (..., N, D), or (N, D) with a radius")
    pdim = _pdim("knn_filter", points, pdim)
    N = points.shape[-2]
    if not isinstance(k, int) or k < 0 or k + 1 > 32 or k + 1 > N:
        raise ValueError(f"knn_filter: k + 1 must be in 1..min(32, N) with N = {N}, got k = {k}")
    if ord not in _ORD:
        raise ValueError(f"knn_filter: ord must be 1, 2 or inf, got {ord}")
    _check_cuda("knn_filter", points)
    query = points
    if radius is not None:
        query = points[_radius_mask(points, pdim, radius, ord, k)]
    idx = knn(query[..., :pdim], points[..., :pdim], k=k + 1, ord=ord).indices      # (..., M, k + 1)
    lead, M, D = idx.shape[:-2], idx.shape[-2], points.shape[-1]
    rows = idx.reshape(*lead, M * (k + 1), 1).expand(*lead, M * (k + 1), D)
    return torch.gather(points.expand(*lead, N, D), -2, rows).view(*lead, M, k + 1, D).mean(dim=-2)
