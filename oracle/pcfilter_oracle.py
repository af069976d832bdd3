"""numpy oracle of the point-cloud filters and svdstf (DESIGN.md §3.5).

Voxel centroids are computed in the input dtype, the way the reference's `index_add_` on the CPU sums them (each voxel's
rows in increasing index order, starting from 0), so they can be compared bit for bit; everything else is fp64.
Test infrastructure only: the package never imports it.
"""
import numpy as np

from oracle import icp_oracle


def voxel_coords(points, voxel):
    """Integer voxel coordinates trunc((p - min) / v) with the sizes rounded to float32 first and a separate subtract and
    divide in the points' dtype."""
    p = np.asarray(points)
    vdim = len(voxel)
    v = np.asarray(voxel, np.float32).astype(p.dtype)
    x = p[:, :vdim]
    return ((x - x.min(0)) / v).astype(np.int64)


def voxel_segments(points, voxel):
    """-> order (rows sorted by voxel, then index), start of every voxel in `order` (M + 1), voxel id of every point."""
    c = voxel_coords(points, voxel)
    order = np.lexsort(c.T[::-1])
    cs = c[order]
    head = np.ones(len(order), bool)
    head[1:] = (cs[1:] != cs[:-1]).any(1)
    start = np.append(np.flatnonzero(head), len(order))
    vid = np.empty(len(order), np.int64)
    vid[order] = np.cumsum(head) - 1
    return order, start, vid


def voxel_centroids(points, voxel):
    """(M, D) centroids in the points' dtype: sequential sums from 0 in index order, divided by the count summed the
    same way (a float32 count stops at 2^24)."""
    p = np.asarray(points)
    order, start, _ = voxel_segments(p, voxel)
    M, D = len(start) - 1, p.shape[1]
    counts = np.diff(start)
    acc = np.zeros((M, D), p.dtype)
    if M and counts.max() <= M:              # few members per voxel: one vectorised step per member rank
        for r in range(int(counts.max())):
            live = np.flatnonzero(counts > r)
            acc[live] += p[order[start[live] + r]]
    else:                                    # few voxels: one sequential accumulate per voxel
        for m in range(M):
            rows = p[order[start[m]:start[m + 1]]]
            acc[m] = np.add.accumulate(np.concatenate([np.zeros((1, D), p.dtype), rows]), axis=0)[-1]
    n = np.minimum(counts, 2 ** 24 if p.dtype == np.float32 else 2 ** 53).astype(p.dtype)
    return acc / n[:, None]


def radius_counts(points, radius, pdim=None, ord=2, chunk=1024):
    """Brute-force count of the points within `radius` (fp64 distances) of every point, itself included."""
    p = np.asarray(points, np.float64)
    p = p[:, :pdim or p.shape[1]]
    out = np.empty(len(p), np.int64)
    for i in range(0, len(p), chunk):
        out[i:i + chunk] = (icp_oracle.distances(p[i:i + chunk], p, ord) <= radius).sum(1)
    return out


def nbr_mask(points, nbr, radius, pdim=None, ord=2):
    return radius_counts(points, radius, pdim, ord) - 1 >= nbr


def knn_filter(points, k, pdim=None, radius=None, ord=2):
    """fp64 knn_filter; with a radius the neighbours of the kept points come from the full cloud."""
    p = np.asarray(points, np.float64)
    pdim = pdim or p.shape[-1]
    q = p if radius is None else p[nbr_mask(p, k, radius, pdim, ord)]
    _, idx = icp_oracle.knn(q[..., :pdim], p[..., :pdim], k + 1, ord)
    return _gather_mean(p, idx)


def _gather_mean(p, idx):
    """rows idx (..., M, k + 1) of p (..., N, D) averaged over the k + 1 neighbours -> (..., M, D)."""
    lead = idx.shape[:-2]
    pb = np.broadcast_to(p, lead + p.shape[-2:])
    flat = idx.reshape(lead + (-1,))
    g = np.take_along_axis(pb, flat[..., None], -2)
    return g.reshape(idx.shape + (p.shape[-1],)).mean(-2)


def svdstf(source, target, with_scale=True):
    """Umeyama in fp64 -> (..., 3, 4) [s R | t]."""
    s, t = np.asarray(source, np.float64), np.asarray(target, np.float64)
    cs, ct = s.mean(-2, keepdims=True), t.mean(-2, keepdims=True)
    s_, t_ = s - cs, t - ct
    H = np.swapaxes(t_, -1, -2) @ s_ / s.shape[-2]
    U, D, Vh = np.linalg.svd(H)
    M = np.broadcast_to(np.eye(3), U.shape).copy()
    M[..., 2, 2] = np.sign(np.linalg.det(U @ Vh))
    if with_scale:
        scale = (np.diagonal(M, axis1=-2, axis2=-1) * D).sum(-1) / (s_ ** 2).sum(-1).mean(-1)
    else:
        scale = np.ones(D.shape[:-1])
    R = U @ M @ Vh
    tr = np.swapaxes(ct, -1, -2) - scale[..., None, None] * R @ np.swapaxes(cs, -1, -2)
    return np.concatenate([scale[..., None, None] * R, tr], -1)
