"""numpy oracle of pp.metric.ape / rpe (DESIGN.md §3.6), with the reference's exact selection rules.

- Association: for each short stamp, searchsorted in the shifted long stamps fl(l + off), the smaller of the two
  bracketing distances |fl(s - l')|, then a walk to the lowest index of equal distances; kept when < diff.
- Distance pairing: segment lengths with the rounding of torch's fp64 3-vector norm on the CPU (taken from torch), a
  sequential cumsum, a binary search per pose with the same tie walk, and the greedy walk with resets.
- Errors follow the reference's formulas in fp64 (lie_oracle for the group operations); statistics use math.fsum and
  the order statistic at (M - 1) // 2.
Test infrastructure only: the package never imports it.
"""
import math

import numpy as np
import torch

from oracle import lie_oracle as L

KEYS = ['Max', 'Min', 'Mean', 'Median', 'RMSE', 'SSE', 'STD']
ETYPES = ['translation', 'rotation', 'pose', 'radian', 'degree']


def associate(rstamp, estamp, diff=0.01, offset=0.0):
    """(r_idx, e_idx) of the matched poses, in increasing short index, and the short length."""
    rs = np.asarray(rstamp, np.float64)
    es = np.asarray(estamp, np.float64)
    snd_longer = len(es) > len(rs)
    short, long_ = (rs, es) if snd_longer else (es, rs)
    off = offset if snd_longer else -offset
    lp = long_ + np.float64(off)
    n = len(lp)
    p = np.searchsorted(lp, short, side='left')
    pl = np.maximum(p - 1, 0)
    pr = np.minimum(p, n - 1)
    dl = np.abs(short - lp[pl])
    dr = np.abs(short - lp[pr])
    right = (p == 0) | ((p < n) & (dr < dl))
    j = np.where(right, pr, pl)
    d = np.where(right, dr, dl)
    walk = ~right
    while True:                     # lowest index among equal distances to the left
        m = walk & (j > 0)
        m[m] = np.abs(short[m] - lp[j[m] - 1]) == d[m]
        if not m.any():
            break
        j[m] -= 1
    keep = d < diff
    si, li = np.nonzero(keep)[0], j[keep]
    r_idx, e_idx = (si, li) if snd_longer else (li, si)
    return r_idx, e_idx, len(short)


def seg_lengths(t):
    """||t_k - t_{k+1}|| for k < N - 1 with the rounding of torch.linalg.norm on fp64 CPU tensors (an FMA chain)."""
    t = torch.from_numpy(np.ascontiguousarray(t, np.float64))
    return torch.linalg.norm(t[:-1] - t[1:], dim=-1).numpy()


def accumulated(t):
    """cat(0, cumsum(l)) with a sequential sum."""
    l = seg_lengths(t)
    D = np.empty(len(l) + 1)
    D[0] = 0.0
    np.cumsum(l, out=D[1:])       # numpy's fp64 cumsum adds left to right
    return D


def pairs_by_dist(t, delta, tol=0.0, all=False):
    t = np.asarray(t, np.float64)
    n = len(t)
    if all:
        D = accumulated(t)
        i = np.arange(n - 1)
        lo, hi = i + 1, np.full(n - 1, n)
        while (lo < hi).any():      # first j > i with fl(D_j - D_i) >= delta
            a = lo < hi
            mid = (lo + hi) // 2
            ge = (D[np.minimum(mid, n - 1)] - D[i]) >= delta
            hi = np.where(a & ge, mid, hi)
            lo = np.where(a & ~ge, mid + 1, lo)
        p = lo
        h = lambda j: np.abs((D[j] - D[i]) - delta)    # noqa: E731
        pl, pr = np.maximum(p - 1, i + 1), np.minimum(p, n - 1)
        hl, hr = h(pl), h(pr)
        right = (p == i + 1) | ((p < n) & (hr < hl))
        j = np.where(right, pr, pl)
        hm = np.where(right, hr, hl)
        walk = ~right
        while True:
            m = walk & (j > i + 1)
            m[m] = np.abs((D[j[m] - 1] - D[i[m]]) - delta) == hm[m]
            if not m.any():
                break
            j[m] -= 1
        ok = ~(hm > tol)
        return i[ok], j[ok]
    l = np.concatenate([[0.0], seg_lengths(t)])
    idx, cur = [], 0.0
    for k in range(n):
        cur += float(l[k])
        if cur >= delta:
            idx.append(k)
            cur = 0.0
    idx = np.asarray(idx, np.int64)
    return idx[:-1], idx[1:]


def pairs_by_frames(n, delta, all=False):
    d = int(delta)
    if all:
        a = np.arange(max(n - d, 0))
        return a, a + d
    ids = np.arange(0, n, d)
    return ids[:-1], ids[1:]


def align(S, poses):
    """Sim3 S [t, q, s] @ Sim3(pose, 1), keeping [t, q]; S None: the poses."""
    P = np.asarray(poses, np.float64)
    if S is None:
        return P
    S = np.broadcast_to(np.asarray(S, np.float64), P.shape[:-1] + (8,))
    X = np.concatenate([P, np.ones(P.shape[:-1] + (1,))], -1)
    return L.mul("Sim3", S, X)[..., :7]


def _mat2so3(R):
    """mat2SO3(check=False) with the reference's branch rule (pypose/lietensor/convert.py:97-145)."""
    m = np.swapaxes(R, -1, -2)
    d2 = m[..., 2, 2] < 1e-5
    d0d1 = m[..., 0, 0] > m[..., 1, 1]
    d0nd1 = m[..., 0, 0] < -m[..., 1, 1]
    t0 = 1 + m[..., 0, 0] - m[..., 1, 1] - m[..., 2, 2]
    q0 = np.stack([m[..., 1, 2] - m[..., 2, 1], t0, m[..., 0, 1] + m[..., 1, 0], m[..., 2, 0] + m[..., 0, 2]], -1)
    t1 = 1 - m[..., 0, 0] + m[..., 1, 1] - m[..., 2, 2]
    q1 = np.stack([m[..., 2, 0] - m[..., 0, 2], m[..., 0, 1] + m[..., 1, 0], t1, m[..., 1, 2] + m[..., 2, 1]], -1)
    t2 = 1 - m[..., 0, 0] - m[..., 1, 1] + m[..., 2, 2]
    q2 = np.stack([m[..., 0, 1] - m[..., 1, 0], m[..., 2, 0] + m[..., 0, 2], m[..., 1, 2] + m[..., 2, 1], t2], -1)
    t3 = 1 + m[..., 0, 0] + m[..., 1, 1] + m[..., 2, 2]
    q3 = np.stack([t3, m[..., 1, 2] - m[..., 2, 1], m[..., 2, 0] - m[..., 0, 2], m[..., 0, 1] - m[..., 1, 0]], -1)
    c = [d2 & d0d1, d2 & ~d0d1, ~d2 & d0nd1, ~d2 & ~d0nd1]
    q = sum(ci[..., None] * qi for ci, qi in zip(c, [q0, q1, q2, q3]))
    t = sum(ci * ti for ci, ti in zip(c, [t0, t1, t2, t3]))
    q = q / (2 * np.sqrt(t))[..., None]
    return q[..., [1, 2, 3, 0]]


def _rot(q):
    """R(q) with columns Act(q, e_j), as matrix() builds it."""
    I = np.broadcast_to(np.eye(3), q.shape[:-1] + (3, 3))
    return np.swapaxes(L.SO3_act(q[..., None, :], I), -1, -2)


def _error(E, etype, t=None):
    if etype == 'translation':
        return np.linalg.norm(E[..., :3] if t is None else t, axis=-1)
    R = _rot(E[..., 3:])
    if etype in ('rotation', 'pose'):
        s = ((R - np.eye(3)) ** 2).sum((-2, -1))
        if etype == 'pose':
            s = s + (E[..., :3] ** 2).sum(-1)
        return np.sqrt(s)
    r = np.linalg.norm(L.SO3_log(_mat2so3(R)), axis=-1)
    return np.rad2deg(r) if etype == 'degree' else r


def ape_errors(r, e, etype):
    """r, e: associated poses, e already aligned."""
    if etype == 'translation':
        return _error(None, etype, e[..., :3] - r[..., :3])
    return _error(L.mul("SE3", L.inv("SE3", e), r), etype)


def rpe_errors(ra, rb, ea, eb, etype):
    Rr = L.mul("SE3", L.inv("SE3", ra), rb)
    Re = L.mul("SE3", L.inv("SE3", ea), eb)
    return _error(L.mul("SE3", L.inv("SE3", Rr), Re), etype)


def stats(err):
    a = np.abs(np.asarray(err, np.float64))
    M = len(a)
    mean = math.fsum(a) / M
    sse = math.fsum(a * a)
    std = math.sqrt(math.fsum((a - mean) ** 2) / (M - 1)) if M > 1 else float('nan')
    return {'Max': a.max(), 'Min': a.min(), 'Mean': mean, 'Median': np.sort(a)[(M - 1) // 2],
            'RMSE': math.sqrt(sse / M), 'SSE': sse, 'STD': std}


def umeyama(src, tgt, with_scale):
    """svdstf in fp64 numpy (geometry.py:361-432)."""
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    cs, ct = src.mean(0), tgt.mean(0)
    s_, t_ = src - cs, tgt - ct
    H = t_.T @ s_ / len(src)
    U, D, V = np.linalg.svd(H)
    M = np.eye(3)
    M[2, 2] = np.sign(np.linalg.det(U @ V))
    sc = (np.diag(M) * D).sum() / (np.linalg.norm(s_, axis=-1) ** 2).mean() if with_scale else 1.0
    R = U @ M @ V
    t = ct - sc * R @ cs
    q = _mat2so3(R)
    return np.concatenate([t, q, [sc]])


def ape(rstamp, rpose, estamp, epose, etype='translation', diff=0.01, offset=0.0, align_=False, scale=False,
        nposes=-1, origin=False):
    """(errors, r_idx, e_idx, S) of APE; nposes means the first nposes associated poses."""
    r_idx, e_idx, _ = associate(rstamp, estamp, diff, offset)
    rp, ep = np.asarray(rpose, np.float64)[r_idx], np.asarray(epose, np.float64)[e_idx]
    S = alignment(rp, ep, align_, scale, nposes, origin)
    return ape_errors(rp, align(S, ep), etype), r_idx, e_idx, S


def alignment(rp, ep, align_, scale, nposes, origin):
    if align_ or scale:
        m = len(rp) if nposes == -1 else nposes
        return umeyama(ep[:m, :3], rp[:m, :3], scale)
    if origin:
        T = L.mul("SE3", rp[:1], L.inv("SE3", ep[:1]))[0]
        return np.concatenate([T, [1.0]])
    return None


def rpe(rstamp, rpose, estamp, epose, etype='translation', diff=0.01, offset=0.0, align_=False, scale=False,
        nposes=-1, origin=False, associate_='frame', delta=1.0, rtol=0.1, all=False, rpair=False):
    """(errors, src, tgt) of RPE; src / tgt index the associated poses."""
    r_idx, e_idx, _ = associate(rstamp, estamp, diff, offset)
    rp, ep = np.asarray(rpose, np.float64)[r_idx], np.asarray(epose, np.float64)[e_idx]
    S = alignment(rp, ep, align_, scale, nposes, origin)
    ea = align(S, ep)
    if associate_ == 'frame':
        src, tgt = pairs_by_frames(len(rp), delta, all)
    else:
        src, tgt = pairs_by_dist((rp if rpair else ea)[:, :3], delta, delta * rtol, all)
    return rpe_errors(rp[src], rp[tgt], ea[src], ea[tgt], etype), src, tgt


# ---------------------------------------------------------------- synthetic inputs of the goldens
# The golden file stores a recipe for each input array instead of its values.  Every recipe is evaluated with integer
# hashing (splitmix64) and correctly rounded elementwise fp64 operations only, so it gives the same bits on every machine.

def _uniform(n, seed):
    """n uniforms in [0, 1) from splitmix64 of (seed, index)."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) * np.uint64(0xD1B54A32D192ED03) + (np.arange(n, dtype=np.uint64) + np.uint64(1)) * \
            np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _unit(q):
    s = q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]
    return q / np.sqrt(s)[:, None]


def synth(recipe, store=None):
    """Evaluate an input recipe (a JSON list):
        ["traj", n, seed, plateaus]          a smooth path with unit quaternions; plateaus: runs of stationary poses
        ["perturb", r, seed, s]              noise of size s on the translations and quaternions (renormalised)
        ["stamps", n, hz, t0, seed, jitter]  t0 + k / hz + jitter u_k
        ["slice", r, start, stop, step]      rows of r
        ["repeat", r, k]                     every row k times
        ["sim3inv", r]                       the fixed Sim3 SIM3_FIXED^-1 applied to the poses r
        ["f32", r]                           r rounded to float32
        ["in", key]                          an array stored in `store` under key
    """
    op, a = recipe[0], recipe[1:]
    if op == "traj":
        n, seed, plateaus = a
        u = _uniform(7 * n, seed).reshape(n, 7)
        step = (u[:, :3] - 0.5) * 0.1 + np.array([0.03, 0.01, 0.0])
        if plateaus:
            step[(np.arange(n) // 7) % 3 == 0] = 0.0
        step[0] = 0.0
        t = np.cumsum(step, 0)
        q = (u[:, 3:] - 0.5) * 0.1 + np.array([0.0, 0.0, 0.0, 1.0])
        return np.concatenate([t, _unit(q)], -1)
    if op == "perturb":
        P = synth(a[0], store)
        u = _uniform(7 * len(P), a[1]).reshape(len(P), 7)
        s = a[2]
        return np.concatenate([P[:, :3] + s * (u[:, :3] - 0.5), _unit(P[:, 3:] + s * (u[:, 3:] - 0.5))], -1)
    if op == "stamps":
        n, hz, t0, seed, jitter = a
        return t0 + np.arange(n, dtype=np.float64) / hz + jitter * _uniform(n, seed)
    if op == "slice":
        return np.ascontiguousarray(synth(a[0], store)[slice(*a[1:])])
    if op == "repeat":
        return np.repeat(synth(a[0], store), a[1], axis=0)
    if op == "sim3inv":
        P = synth(a[0], store)
        S = L.inv("Sim3", SIM3_FIXED[None])
        return align(S[0], P)
    if op == "f32":
        return synth(a[0], store).astype(np.float32)
    if op == "in":
        return np.asarray(store[a[0]])
    raise ValueError(recipe)


SIM3_FIXED = np.array([0.5, -1.0, 0.3, 0.1, 0.2, -0.1, 0.9695359714832659, 1.7])
SIM3_FIXED[3:7] /= np.sqrt((SIM3_FIXED[3:7] * SIM3_FIXED[3:7]).sum())
