"""CPU oracle of the LM inner loop — TEST INFRASTRUCTURE ONLY (see lie_oracle.py header).

Restates pypose/optim/optimizer.py:645-680 (dense LevenbergMarquardt.step) in numpy, twice:

* `dense_lm_step`  — literally the reference algorithm on a dense Jacobian with 7 columns per SE3 pose
  (the 7th identically zero, optimizer.py:657 clamp making its diagonal 1e-6, SURVEY.md §3.3);
* block functions (`poseinv_trial`, `reproj_accum`, `solve6_retract`, ...) with the C-ABI signatures
  of csrc/lm.cu, which are what the CUDA kernels are compared against.

tests/test_lm.py checks block == dense, and both against trajectories recorded from the reference's
own LM (tests/golden/lm.npz, oracle/make_golden_lm.py).
"""
import math
from fractions import Fraction

import numpy as np

from . import lie_oracle as O


def _triu_pack(A):
    iu = np.triu_indices(6)
    return A[..., iu[0], iu[1]]


def _triu_unpack(H21):
    iu = np.triu_indices(6)
    A = np.zeros(H21.shape[:-1] + (6, 6), dtype=H21.dtype)
    A[..., iu[0], iu[1]] = H21
    A[..., iu[1], iu[0]] = H21
    return A


# ------------------------------------------------------------------ robust kernels + FastTriggs
def robust(kind, delta, x):
    """rho(x), rho'(x) for pypose/optim/kernel.py (Huber :5-45, PseudoHuber :48-86, Cauchy :89-126,
    SoftLOne :129-168, Arctan :171-207, Scale :258-297); FastTriggs scales R and J rows by sqrt(rho')
    (corrector.py:73-95)."""
    d2 = delta * delta
    with np.errstate(all="ignore"):
        if kind == 1:
            root = np.sqrt(x)
            return np.where(root < delta, x, 2 * delta * root - d2), np.where(root < delta, 1.0, delta / root)
        if kind == 2:
            q = np.sqrt(x / d2 + 1)
            return 2 * d2 * (q - 1), 1 / q
        if kind == 3:
            q = x / d2 + 1
            return d2 * np.log(q), 1 / q
        if kind == 4:
            q = np.sqrt(1 / d2 + x)
            return 2 * (delta * q - 1), delta / q
        if kind == 5:
            q = x / d2
            return d2 * np.arctan(q), 1 / (1 + q * q)
        if kind == 6:
            return delta * x, np.full_like(x, delta)
    return x, np.ones_like(x)


# ------------------------------------------------------------------ PoseInv: r = Log(P X)
def poseinv_residual(P, X):
    return O.log("SE3", O.mul("SE3", P, X))


def poseinv_jac_blocks(P, X):
    """d Log(P X) / dP (left perturbation) = Jl^-1(r): the reference obtains it as the product of
    SE3_Log.backward (op.py:389-395) and SE3_Mul.backward wrt X (identity, op.py:870-877)."""
    r = poseinv_residual(P, X)
    return r, O.se3_Jl_inv(r)


def damped_solve(A, g, scale, dmin, dmax):
    """clamp (optimizer.py:657), cumulative damping (:666), Cholesky solve (solver.py:213-216)."""
    A0 = A.copy()
    A = A.copy()
    idx = np.arange(A.shape[-1])
    A[..., idx, idx] = np.clip(A[..., idx, idx], dmin, dmax) * scale
    L = np.linalg.cholesky(A)
    y = np.linalg.solve(L, -g[..., None])
    D = np.linalg.solve(np.swapaxes(L, -1, -2), y)[..., 0]
    predicted = np.einsum('...i,...ij,...j->...', D, A0, D) + 2 * np.einsum('...i,...i->...', D, g)
    return D, predicted


def retract(D, P):
    return O.mul("SE3", O.exp("SE3", D), P)


def poseinv_loss(P, X, kind=0, delta=1.0):
    return np.array([robust(kind, delta, (poseinv_residual(P, X) ** 2).sum(-1))[0].sum()])


def poseinv_trial(P, X, scale, dmin, dmax, kind=0, delta=1.0):
    r, J = poseinv_jac_blocks(P, X)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    A = np.swapaxes(J, -1, -2) @ J * w[:, None, None]
    g = (np.swapaxes(J, -1, -2) @ r[..., None])[..., 0] * w[:, None]
    D, pred = damped_solve(A, g, scale, dmin, dmax)
    Pt = retract(D, P)
    rho_t, _ = robust(kind, delta, (poseinv_residual(Pt, X) ** 2).sum(-1))
    return Pt, np.array([rho.sum(), rho_t.sum(), pred.sum(), 0.0])


# ------------------------------------------------------------------ Reproj: r = pi(T p) - z
def reproj_residual(poses, pts, pix, cidx):
    y = O.act("SE3", poses[cidx], pts)
    return -y[:, :2] / y[:, 2:] - pix


def reproj_jac_rows(poses, pts, cidx):
    """(m, 2, 6): d pi/dy @ [I, -y^]  (SE3_Act_Jacobian, op.py:225-227, applied to out = T p)."""
    y = O.act("SE3", poses[cidx], pts)
    m = y.shape[0]
    dpi = np.zeros((m, 2, 3))
    dpi[:, 0, 0] = -1 / y[:, 2]
    dpi[:, 1, 1] = -1 / y[:, 2]
    dpi[:, 0, 2] = y[:, 0] / y[:, 2] ** 2
    dpi[:, 1, 2] = y[:, 1] / y[:, 2] ** 2
    dy = np.concatenate([np.broadcast_to(np.eye(3), (m, 3, 3)), O.vec2skew(-y)], -1)
    return dpi @ dy


def reproj_accum(poses, pts, pix, seg, kind=0, delta=1.0):
    C = poses.shape[0]
    cidx = np.repeat(np.arange(C), np.diff(seg))
    r = reproj_residual(poses, pts, pix, cidx)
    J = reproj_jac_rows(poses, pts, cidx)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    A = np.zeros((C, 6, 6))
    g = np.zeros((C, 6))
    np.add.at(A, cidx, np.swapaxes(J, -1, -2) @ J * w[:, None, None])
    np.add.at(g, cidx, (np.swapaxes(J, -1, -2) @ r[..., None])[..., 0] * w[:, None])
    return _triu_pack(A), g, np.array([rho.sum()])


def seg_sum(x, seg):
    """Row sums of x per segment [seg[c], seg[c+1]) of rows sorted by segment: np.add.reduceat over the non-empty
    segments (reduceat alone returns the next row for an empty one); an empty segment sums to 0."""
    seg = np.asarray(seg, dtype=np.int64)
    out = np.zeros((seg.size - 1,) + x.shape[1:], dtype=np.float64)
    ne = np.flatnonzero(seg[1:] > seg[:-1])
    if ne.size:
        out[ne] = np.add.reduceat(x[:seg[-1]], seg[ne], axis=0)
    return out


def reproj_accum_seg(poses, pts, pix, seg, kind=0, delta=1.0):
    """reproj_accum per camera with a segment reduction over the camera-sorted rows instead of np.add.at (fast at
    1e6 rows): (C, 21) H, (C, 6) g and the (C,) loss of each camera."""
    C = poses.shape[0]
    m = int(seg[-1])
    cidx = np.repeat(np.arange(C), np.diff(seg))
    r = reproj_residual(poses, pts[:m], pix[:m], cidx)
    J = reproj_jac_rows(poses, pts[:m], cidx)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    iu = np.triu_indices(6)
    JJ = np.einsum('mka,mkb->mab', J, J)[:, iu[0], iu[1]] * w[:, None]
    Jr = np.einsum('mka,mk->ma', J, r) * w[:, None]
    return seg_sum(JJ, seg), seg_sum(Jr, seg), seg_sum(rho, seg)


def damped_solve_flagged(A, g, scale, dmin, dmax):
    """damped_solve per block with a per-block failure flag instead of the exception np.linalg.cholesky raises for the
    whole batch: (D, predicted, failed), D = 0 and predicted = 0 on the blocks whose damped matrix is not positive
    definite."""
    idx = np.arange(A.shape[-1])
    Ad = A.copy()
    Ad[..., idx, idx] = np.clip(Ad[..., idx, idx], dmin, dmax) * scale
    failed = np.linalg.eigvalsh(Ad)[..., 0] <= 0
    D, pred = np.zeros(g.shape), np.zeros(g.shape[:-1])
    ok = ~failed
    if ok.any():
        D[ok], pred[ok] = damped_solve(A[ok], g[ok], scale, dmin, dmax)
    return D, pred, failed


def solve6_retract(H21, g, P, scale, dmin, dmax):
    D, pred = damped_solve(_triu_unpack(H21), g, scale, dmin, dmax)
    return retract(D, P), D, np.array([pred.sum(), 0.0])


def reproj_loss(poses, pts, pix, cidx, kind=0, delta=1.0):
    return np.array([robust(kind, delta, (reproj_residual(poses, pts, pix, cidx) ** 2).sum(-1))[0].sum()])


# ------------------------------------------------------------------ PGO: r = Log(Z^-1 A^-1 B)
def pgo_residual(nodes, Z, ei, ej):
    """examples/module/pgo/pgo.py:21-25."""
    S = O.mul("SE3", O.inv("SE3", Z), O.inv("SE3", nodes[ei]))
    return O.log("SE3", O.mul("SE3", S, nodes[ej])), S


def pgo_jac_blocks(nodes, Z, ei, ej, exact=False):
    """d r / d B = Jl^-1(r) Adj(Z^-1 A^-1) (SE3_Log.backward op.py:389-395 chained with SE3_Mul.backward wrt Y
    op.py:870-877); d r / d A = -(that) (SE3_Inv.backward op.py:968-973 + SE3_Mul.backward wrt X).
    exact=True: Jl^-1 from se3_Jl_inv_exact instead of the reference's closed forms."""
    r, S = pgo_residual(nodes, Z, ei, ej)
    return r, (se3_Jl_inv_exact(r) if exact else O.se3_Jl_inv(r)) @ O.SE3_Adj(S)


def _series(th2, coef):
    """sum_n coef[n] th2^n (Horner)."""
    out = np.zeros_like(th2)
    for c in coef[::-1]:
        out = out * th2 + c
    return out


_FACT = [float(math.factorial(k)) for k in range(40)]
# coefficients in theta^2 of the functions of theta in Jl^-1 (op.py:23-32) and Q (op.py:37-58), to theta^24
def _bernoulli(n):
    """B_0 .. B_n as exact fractions (B_1 = -1/2)."""
    B = [Fraction(1)]
    for m in range(1, n + 1):
        B.append(-sum(math.comb(m + 1, k) * B[k] for k in range(m)) / (m + 1))
    return B


_JLINV_SERIES = [float(abs(b) / math.factorial(2 * n)) for n, b in enumerate(_bernoulli(28)[2::2], 1)]   # B_2n / (2n)!
_Q1_SERIES = [(-1) ** n / _FACT[2 * n + 3] for n in range(13)]        # (th - sin th) / th^3
_Q2_SERIES = [(-1) ** n / _FACT[2 * n + 4] for n in range(13)]        # (th^2 + 2 cos th - 2) / (2 th^4)
_Q3_SERIES = [(-1) ** k * (k - 1) / _FACT[2 * k + 1] for k in range(2, 15)]   # (2 th - 3 sin th + th cos th) / (2 th^5)


def se3_Jl_inv_exact(x):
    """se3 Jl^-1 (lie_oracle.se3_Jl_inv) with every coefficient accurate to a few ulps at every angle: the power series
    below theta = 1, where the closed forms lose up to ~u / theta^4 to cancellation (1e-8 relative at theta = 1e-2 in
    fp64), the closed forms above it."""
    tau, phi = x[..., :3], x[..., 3:]
    th2 = (phi ** 2).sum(-1)[..., None, None]
    th = np.sqrt(th2)
    sm = th < 1.0
    with np.errstate(all="ignore"):
        c = np.where(sm, _series(th2, _JLINV_SERIES), (1 - th * np.cos(th / 2) / (2 * np.sin(th / 2))) / th2)
        c1 = np.where(sm, _series(th2, _Q1_SERIES), (th - np.sin(th)) / (th2 * th))
        c2 = np.where(sm, _series(th2, _Q2_SERIES), (th2 + 2 * np.cos(th) - 2) / (2 * th2 * th2))
        c3 = np.where(sm, _series(th2, _Q3_SERIES), (2 * th - 3 * np.sin(th) + th * np.cos(th)) / (2 * th2 * th2 * th))
    P, T = O.vec2skew(phi), O.vec2skew(tau)
    Ji = np.eye(3) - 0.5 * P + c * (P @ P)
    Q = (0.5 * T + c1 * (P @ T + T @ P + P @ T @ P) + c2 * (P @ P @ T + T @ P @ P - 3 * P @ T @ P)
         + c3 * (P @ T @ P @ P + P @ P @ T @ P))
    Z = np.zeros_like(Ji)
    return np.concatenate([np.concatenate([Ji, -Ji @ Q @ Ji], -1), np.concatenate([Z, Ji], -1)], -2)


def pgo_linearize(nodes, Z, ei, ej, kind=0, delta=1.0, W=None):
    """Per-edge J^T J / J^T r (optimizer.py:654-656).  With information matrices W ((E,6,6) or (1,6,6); `weight` of
    LM.step, normalize_RWJ optimizer.py:80-95) returns (J^T W J, J^T W r, J^T J, J^T r, cost): the unweighted pair is
    what the step-quality term uses (strategy.py:143 receives J and R, not the weight)."""
    r, J = pgo_jac_blocks(nodes, Z, ei, ej)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    Jt = np.swapaxes(J, -1, -2)
    M = Jt @ J * w[:, None, None]
    u = (Jt @ r[..., None])[..., 0] * w[:, None]
    if W is None:
        return _triu_pack(M), u, np.array([rho.sum()])
    W = np.broadcast_to(W.reshape(-1, 6, 6), J.shape)
    Mw = Jt @ W @ J * w[:, None, None]
    uw = (Jt @ W @ r[..., None])[..., 0] * w[:, None]
    return _triu_pack(Mw), uw, _triu_pack(M), u, np.array([rho.sum()])


def pgo_scatter(M21, u, ei, ej, n):
    Hd, g = np.zeros((n, 21)), np.zeros((n, 6))
    np.add.at(Hd, ei, M21); np.add.at(Hd, ej, M21)
    np.add.at(g, ei, -u); np.add.at(g, ej, u)
    return Hd, g


def pgo_spmv(M21, ei, ej, x, y0):
    v = (_triu_unpack(M21) @ (x[ei] - x[ej])[..., None])[..., 0]
    y = y0.copy()
    np.add.at(y, ei, v); np.add.at(y, ej, -v)
    return y


def pgo_loss(nodes, Z, ei, ej, kind=0, delta=1.0):
    return np.array([robust(kind, delta, (pgo_residual(nodes, Z, ei, ej)[0] ** 2).sum(-1))[0].sum()])


def pgo_dense_jac(nodes, Z, ei, ej):
    """The reference's dense (6E, 7N) Jacobian of the PoseGraph model."""
    _, J = pgo_jac_blocks(nodes, Z, ei, ej)
    E, N = len(ei), nodes.shape[0]
    D = np.zeros((6 * E, 7 * N))
    for e in range(E):
        D[6 * e:6 * e + 6, 7 * ei[e]:7 * ei[e] + 6] -= J[e]
        D[6 * e:6 * e + 6, 7 * ej[e]:7 * ej[e] + 6] += J[e]
    return D


# ------------------------------------------------------------------ bundle adjustment: poses AND points are parameters
def ba_residual(poses, points, pix, cidx, pidx):
    """README.md:170-178: project(points[pidx], poses[cidx]) - observations."""
    y = O.act("SE3", poses[cidx], points[pidx])
    return -y[:, :2] / y[:, 2:] - pix


def ba_jac_rows(poses, points, cidx, pidx):
    """Jc (m,2,6) as reproj_jac_rows; Jp (m,2,3) = d pi/dy @ R(T) (SE3_Act.backward wrt p, op.py:560-568)."""
    y = O.act("SE3", poses[cidx], points[pidx])
    m = y.shape[0]
    dpi = np.zeros((m, 2, 3))
    dpi[:, 0, 0] = -1 / y[:, 2]
    dpi[:, 1, 1] = -1 / y[:, 2]
    dpi[:, 0, 2] = y[:, 0] / y[:, 2] ** 2
    dpi[:, 1, 2] = y[:, 1] / y[:, 2] ** 2
    dy = np.concatenate([np.broadcast_to(np.eye(3), (m, 3, 3)), O.vec2skew(-y)], -1)
    return dpi @ dy, dpi @ O.SO3_Adj(poses[cidx][:, 3:])


def ba_linearize(poses, points, pix, cidx, pidx, kind=0, delta=1.0):
    r = ba_residual(poses, points, pix, cidx, pidx)
    Jc, Jp = ba_jac_rows(poses, points, cidx, pidx)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    sw = np.sqrt(w)
    Jc, Jp, rs = Jc * sw[:, None, None], Jp * sw[:, None, None], r * sw[:, None]
    C, P = poses.shape[0], points.shape[0]
    iu = np.triu_indices(3)
    Hcc = _group_sum(cidx, _triu_pack(np.swapaxes(Jc, -1, -2) @ Jc), C)
    Hpp = _group_sum(pidx, (np.swapaxes(Jp, -1, -2) @ Jp)[:, iu[0], iu[1]], P)
    gc = _group_sum(cidx, (np.swapaxes(Jc, -1, -2) @ rs[..., None])[..., 0], C)
    gp = _group_sum(pidx, (np.swapaxes(Jp, -1, -2) @ rs[..., None])[..., 0], P)
    return Jc.reshape(-1, 12), Jp.reshape(-1, 6), rs, Hcc, Hpp, gc, gp, np.array([rho.sum()])


def ba_wtx(Jc, Jp, cidx, pidx, x, npts):
    v = (Jc.reshape(-1, 2, 6) @ x[cidx][..., None])
    t = np.zeros((npts, 3))
    np.add.at(t, pidx, (np.swapaxes(Jp.reshape(-1, 2, 3), -1, -2) @ v)[..., 0])
    return t


def ba_wv(Jc, Jp, cidx, pidx, v, ncam):
    u = (Jp.reshape(-1, 2, 3) @ v[pidx][..., None])
    y = np.zeros((ncam, 6))
    np.add.at(y, cidx, (np.swapaxes(Jc.reshape(-1, 2, 6), -1, -2) @ u)[..., 0])
    return y


def ba_loss(poses, points, pix, cidx, pidx, kind=0, delta=1.0):
    return np.array([robust(kind, delta, (ba_residual(poses, points, pix, cidx, pidx) ** 2).sum(-1))[0].sum()])


def ba_dense_lm_step(poses, points, pix, cidx, pidx, damping, dmin=1e-6, dmax=1e32, reject=16, last=None):
    """optimizer.py:645-680 on the dense (2m, 7C + 3P) Jacobian, parameters ordered [poses, points_3d]."""
    C, P, m = poses.shape[0], points.shape[0], len(cidx)
    R = ba_residual(poses, points, pix, cidx, pidx).reshape(-1)
    Jc, Jp = ba_jac_rows(poses, points, cidx, pidx)
    J = np.zeros((2 * m, 7 * C + 3 * P))
    for k in range(m):
        J[2 * k:2 * k + 2, 7 * cidx[k]:7 * cidx[k] + 6] = Jc[k]
        J[2 * k:2 * k + 2, 7 * C + 3 * pidx[k]:7 * C + 3 * pidx[k] + 3] = Jp[k]
    A = J.T @ J
    d = np.arange(A.shape[0])
    A[d, d] = np.clip(A[d, d], dmin, dmax)
    loss = last = (R ** 2).sum() if last is None else last
    rej = 0
    while last <= loss:
        A[d, d] += A[d, d] * damping
        L_ = np.linalg.cholesky(A)
        D = np.linalg.solve(L_.T, np.linalg.solve(L_, -(J.T @ R)))
        Pn = retract(D[:7 * C].reshape(C, 7)[:, :6], poses)
        pn = points + D[7 * C:].reshape(P, 3)
        loss = (ba_residual(Pn, pn, pix, cidx, pidx) ** 2).sum()
        if last < loss and rej < reject:
            loss, rej = last, rej + 1
        else:
            poses, points = Pn, pn
            break
    return poses, points, loss, last, rej


# ------------------------------------------------------------------ the dense reference algorithm
def dense_lm_step(residual_fn, jac_fn, P, damping, dmin=1e-6, dmax=1e32, reject=16, last=None, update=None):
    """One LevenbergMarquardt.step with a constant damping (optimizer.py:645-680) on parameters P (N,7).

    residual_fn(P) -> R (M,);  jac_fn(P) -> dense J (M, 7N) in the reference's column layout.
    Returns (P_new, loss, last, reject_count)."""
    R = residual_fn(P)
    J = jac_fn(P)
    A = J.T @ J
    d = np.arange(A.shape[0])
    A[d, d] = np.clip(A[d, d], dmin, dmax)
    loss = last = (R ** 2).sum() if last is None else last
    rej = 0
    while last <= loss:
        A[d, d] += A[d, d] * damping
        L = np.linalg.cholesky(A)
        D = np.linalg.solve(L.T, np.linalg.solve(L, -(J.T @ R)))
        Pn = retract(D.reshape(-1, 7)[:, :6], P)
        loss = (residual_fn(Pn) ** 2).sum()
        if last < loss and rej < reject:
            loss, rej = last, rej + 1
        else:
            P = Pn
            break
    return P, loss, last, rej


def dense_jac_from_blocks(blocks, row_param, n_params):
    """Assemble the reference's dense (M*d, 7*N) Jacobian from per-residual (d,6) blocks."""
    m, d, _ = blocks.shape
    J = np.zeros((m * d, 7 * n_params))
    for k in range(m):
        J[k * d:(k + 1) * d, 7 * row_param[k]:7 * row_param[k] + 6] = blocks[k]
    return J


# ------------------------------------------------------------------ two-pose reprojection: r = proj(T_b^-1 T_a p) - z
# (README.md:170-178 project with intr = (-1, 0, 0, -1, 0); function/geometry.py:60-112,171-225 point2pixel / reprojerr
# with K -> intr = (K00, K01, K02, K11, K12); generalises examples/module/reprojpgo/reprojpgo.py:16-28)
README_INTR = (-1.0, 0.0, 0.0, -1.0, 0.0)


def reproj2_residual(nodes, pts, pix, ia, ib, intr=README_INTR):
    fx, sk, cx, fy, cy = intr
    Trel = O.mul("SE3", O.inv("SE3", nodes[ib]), nodes[ia])
    y = O.act("SE3", Trel, pts)
    u = (fx * y[:, 0] + sk * y[:, 1]) / y[:, 2] + cx
    v = fy * y[:, 1] / y[:, 2] + cy
    return np.stack([u, v], -1) - pix, y


def reproj2_jac_rows(nodes, pts, ia, ib, intr=README_INTR):
    """(m, 2, 6) J = d r / d xi_a = d proj/dy @ [I, -y^] @ Adj(T_b^-1) (SE3_Act_Jacobian op.py:225-227, SE3_Mul.backward
    wrt Y op.py:870-877); d r / d xi_b = -J (SE3_Inv.backward op.py:968-973)."""
    fx, sk, cx, fy, cy = intr
    _, y = reproj2_residual(nodes, pts, np.zeros((len(ia), 2)), ia, ib, intr)
    m = y.shape[0]
    dpi = np.zeros((m, 2, 3))
    dpi[:, 0, 0] = fx / y[:, 2]
    dpi[:, 0, 1] = sk / y[:, 2]
    dpi[:, 0, 2] = -(fx * y[:, 0] + sk * y[:, 1]) / y[:, 2] ** 2
    dpi[:, 1, 1] = fy / y[:, 2]
    dpi[:, 1, 2] = -fy * y[:, 1] / y[:, 2] ** 2
    dy = np.concatenate([np.broadcast_to(np.eye(3), (m, 3, 3)), O.vec2skew(-y)], -1)
    return dpi @ dy @ O.SE3_Adj(O.inv("SE3", nodes[ib]))


def reproj2_accum(nodes, pts, pix, pseg, pa, pb, intr=README_INTR, kind=0, delta=1.0):
    """Per ordered pose pair: M (E,21) = sum J^T J, u (E,6) = sum J^T r, cost (1,) — the C-ABI of b200_lm_reproj2_accum."""
    E = len(pa)
    pe = np.repeat(np.arange(E), np.diff(pseg))
    ia, ib = np.asarray(pa)[pe], np.asarray(pb)[pe]
    r, _ = reproj2_residual(nodes, pts, pix, ia, ib, intr)
    J = reproj2_jac_rows(nodes, pts, ia, ib, intr)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    A, g = np.zeros((E, 6, 6)), np.zeros((E, 6))
    np.add.at(A, pe, np.swapaxes(J, -1, -2) @ J * w[:, None, None])
    np.add.at(g, pe, (np.swapaxes(J, -1, -2) @ r[..., None])[..., 0] * w[:, None])
    return _triu_pack(A), g, np.array([rho.sum()])


def reproj2_loss(nodes, pts, pix, ia, ib, intr=README_INTR, kind=0, delta=1.0):
    return np.array([robust(kind, delta, (reproj2_residual(nodes, pts, pix, ia, ib, intr)[0] ** 2).sum(-1))[0].sum()])


def reproj2_dense_jac(nodes, pts, ia, ib, intr=README_INTR):
    """The reference's dense (2m, 7N) Jacobian of the model."""
    J = reproj2_jac_rows(nodes, pts, ia, ib, intr)
    m, N = len(ia), nodes.shape[0]
    D = np.zeros((2 * m, 7 * N))
    for k in range(m):
        D[2 * k:2 * k + 2, 7 * ia[k]:7 * ia[k] + 6] += J[k]
        D[2 * k:2 * k + 2, 7 * ib[k]:7 * ib[k] + 6] -= J[k]
    return D


# ------------------------------------------------------------------ error scales of the linearisations (sum of |term|)
# A kernel that computes an entry as a sum of products in a dtype with unit roundoff u is off by at most about
# u * (the sum of the absolute values of those products).  The *_terms companions return that sum per output entry.  Each
# factor enters with its own such scale, obtained by evaluating the factor's formula on absolute values: a translation
# R^T (t_b - t_a) is counted as |R^T| (|t_b| + |t_a|), a projection's numerator fx y.x + sk y.y as |fx| |y.x| + |sk| |y.y|,
# and a robust weight with its relative sensitivity 2 |r|_abs / delta to the rounding of |r|^2 (kinds 1-5).
def _rot(q):
    return O.SO3_Adj(q)


def _abs_skew(v):
    return np.abs(O.vec2skew(v))


def _group_sum(idx, vals, n):
    """Row sums of vals per value of idx (np.bincount per column: fast at 1e6 rows)."""
    vals = vals.reshape(len(idx), int(np.prod(vals.shape[1:])))
    return np.stack([np.bincount(idx, weights=vals[:, q], minlength=n) for q in range(vals.shape[1])], 1)


def _weight_factor(kind, delta, rabs):
    if kind in (1, 2, 3, 4, 5):
        return 1.0 + 2.0 * np.sqrt((rabs ** 2).sum(-1)) / delta
    return np.ones(rabs.shape[0])


def _rho_terms(kind, delta, x):
    """Sum of |term| of rho(x) itself: PseudoHuber 2 d^2 (q - 1) and SoftLOne 2 (d q - 1) cancel to O(x) from O(1) terms."""
    if kind == 2:
        return 2 * delta * delta * (np.sqrt(x / delta ** 2 + 1) + 1)
    if kind == 4:
        return 2 * (delta * np.sqrt(1 / delta ** 2 + x) + 1)
    return np.abs(robust(kind, delta, x)[0])


def rows_linearize(J, r, grp, n, kind=0, delta=1.0, W=None):
    """M (n, 21) = sum w J^T W J, u (n, 6) = sum w J^T W r and the cost sum rho(|r|^2) over the residual rows (J (m, d, 6),
    r (m, d), information matrices W (m, d, d) or None) grouped by grp into n blocks: the assembly of pgo_linearize /
    reproj2_accum for Jacobians computed once."""
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    WJ = J if W is None else W @ J
    Wr = r if W is None else (W @ r[..., None])[..., 0]
    iu = np.triu_indices(6)
    M = np.einsum('mka,mkb->mab', J, WJ)[:, iu[0], iu[1]] * w[:, None]
    u = np.einsum('mka,mk->ma', J, Wr) * w[:, None]
    return _group_sum(grp, M, n), _group_sum(grp, u, n), np.array([rho.sum()])


def rows_terms(J, r, Jabs, rabs, grp, n, kind=0, delta=1.0, W=None):
    """Sum of |term| of M (n, 21) = sum w J^T J, u (n, 6) = sum w J^T r and the cost sum rho(|r|^2) over the residual rows
    (J (m, d, 6), r (m, d)) grouped by grp into n blocks, from the magnitudes Jabs / rabs of the factors."""
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    ww = w * _weight_factor(kind, delta, rabs)
    iu = np.triu_indices(6)
    WJ = Jabs if W is None else np.abs(W) @ Jabs
    Wr = rabs if W is None else (np.abs(W) @ rabs[..., None])[..., 0]
    MM = np.einsum('mka,mkb->mab', Jabs, WJ)[:, iu[0], iu[1]] * ww[:, None]
    uu = np.einsum('mka,mk->ma', Jabs, Wr) * ww[:, None]
    cost = _rho_terms(kind, delta, (r ** 2).sum(-1)).sum() + (w * 2 * (np.abs(r) * rabs).sum(-1)).sum()
    return _group_sum(grp, MM, n), _group_sum(grp, uu, n), np.array([cost])


def pgo_terms(nodes, Z, ei, ej):
    """Magnitudes (Jabs (E,6,6), rabs (E,6)) of the factors of pgo_jac_blocks."""
    r, S = pgo_residual(nodes, Z, ei, ej)
    A, B = nodes[ei], nodes[ej]
    RZt, RAt = np.swapaxes(_rot(Z[:, 3:]), -1, -2), np.swapaxes(_rot(A[:, 3:]), -1, -2)
    tabs = (np.abs(RZt) @ ((np.abs(RAt) @ (np.abs(B[:, :3]) + np.abs(A[:, :3]))[..., None])[..., 0] + np.abs(Z[:, :3]))[..., None])[..., 0]
    rabs = np.concatenate([(np.abs(O.so3_Jl_inv(r[:, 3:])) @ tabs[..., None])[..., 0], np.abs(r[:, 3:]) + 1.0], -1)
    # R_S = R_Z^T R_A^T R_B and the rotation of r come from products of unit quaternions: their entries carry O(1) terms
    # even where the residual rotation is small
    Jl = np.abs(O.se3_Jl_inv(r))
    Jl[:, :3, 3:] += _abs_skew(rabs[:, :3])
    for k in (slice(0, 3), slice(3, 6)):
        Jl[:, k, k] += 0.5 * _abs_skew(rabs[:, 3:])
    RS = np.abs(np.swapaxes(_rot(Z[:, 3:]), -1, -2)) @ np.abs(RAt) @ np.abs(_rot(B[:, 3:]))
    AdjA = np.concatenate([np.concatenate([RS, _abs_skew(tabs) @ RS], -1),
                           np.concatenate([np.zeros_like(RS), RS], -1)], -2)
    return Jl @ AdjA, rabs


def pgo_linearize_terms(nodes, Z, ei, ej, kind=0, delta=1.0, W=None):
    """Sum of |term| of each output of pgo_linearize (per edge; with W the weighted pair first, as pgo_linearize)."""
    r, J = pgo_jac_blocks(nodes, Z, ei, ej)
    Jabs, rabs = pgo_terms(nodes, Z, ei, ej)
    E = len(ei)
    M, u, cost = rows_terms(J, r, Jabs, rabs, np.arange(E), E, kind, delta)
    if W is None:
        return M, u, cost
    Mw, uw, _ = rows_terms(J, r, Jabs, rabs, np.arange(E), E, kind, delta, np.broadcast_to(W.reshape(-1, 6, 6), J.shape))
    return Mw, uw, M, u, cost


def _proj_abs(y, yabs, intr):
    """Magnitudes of d proj / d y (m,2,3) and of proj(y) (m,2) for intrinsics (fx, sk, cx, fy, cy)."""
    fx, sk, cx, fy, cy = (abs(v) for v in intr)
    z = np.abs(y[:, 2])
    zf = yabs[:, 2] / z                                     # the rounding of 1 / y.z, relative
    m = len(y)
    d = np.zeros((m, 2, 3))
    d[:, 0, 0], d[:, 0, 1] = fx / z, sk / z
    d[:, 0, 2] = (fx * yabs[:, 0] + sk * yabs[:, 1]) / z ** 2
    d[:, 1, 1], d[:, 1, 2] = fy / z, fy * yabs[:, 1] / z ** 2
    p = np.stack([(fx * yabs[:, 0] + sk * yabs[:, 1]) / z + cx, fy * yabs[:, 1] / z + cy], -1)
    return d * zf[:, None, None], p * zf[:, None]


def reproj2_terms(nodes, pts, pix, ia, ib, intr=README_INTR):
    """Magnitudes (Jabs (m,2,6), rabs (m,2)) of the factors of reproj2_jac_rows / reproj2_residual."""
    _, y = reproj2_residual(nodes, pts, pix, ia, ib, intr)
    Ta, Tb = nodes[ia], nodes[ib]
    Ra, Rbt = np.abs(_rot(Ta[:, 3:])), np.abs(np.swapaxes(_rot(Tb[:, 3:]), -1, -2))
    wabs = (Ra @ np.abs(pts)[..., None])[..., 0] + np.abs(Ta[:, :3])
    yabs = (Rbt @ (wabs + np.abs(Tb[:, :3]))[..., None])[..., 0]
    dpi, pabs = _proj_abs(y, yabs, intr)
    tinv = (Rbt @ np.abs(Tb[:, :3])[..., None])[..., 0]
    Adj = np.concatenate([np.concatenate([Rbt, _abs_skew(tinv) @ Rbt], -1),
                          np.concatenate([np.zeros_like(Rbt), Rbt], -1)], -2)
    dy = np.concatenate([np.broadcast_to(np.eye(3), (len(y), 3, 3)), _abs_skew(yabs)], -1)
    return dpi @ dy @ Adj, pabs + np.abs(pix)


def reproj2_accum_terms(nodes, pts, pix, pseg, pa, pb, intr=README_INTR, kind=0, delta=1.0):
    """Sum of |term| of each output of reproj2_accum (per pair)."""
    E = len(pa)
    pe = np.repeat(np.arange(E), np.diff(pseg))
    ia, ib = np.asarray(pa)[pe], np.asarray(pb)[pe]
    r, _ = reproj2_residual(nodes, pts, pix, ia, ib, intr)
    J = reproj2_jac_rows(nodes, pts, ia, ib, intr)
    Jabs, rabs = reproj2_terms(nodes, pts, pix, ia, ib, intr)
    return rows_terms(J, r, Jabs, rabs, pe, E, kind, delta)


def ba_terms(poses, points, pix, cidx, pidx):
    """Magnitudes (Jc_abs (m,2,6), Jp_abs (m,2,3), rabs (m,2)) of the factors of ba_jac_rows / ba_residual."""
    y = O.act("SE3", poses[cidx], points[pidx])
    R = np.abs(_rot(poses[cidx][:, 3:]))
    yabs = (R @ np.abs(points[pidx])[..., None])[..., 0] + np.abs(poses[cidx][:, :3])
    dpi, pabs = _proj_abs(y, yabs, README_INTR)
    dy = np.concatenate([np.broadcast_to(np.eye(3), (len(y), 3, 3)), _abs_skew(yabs)], -1)
    return dpi @ dy, dpi @ R, pabs + np.abs(pix)


def ba_linearize_terms(poses, points, pix, cidx, pidx, kind=0, delta=1.0):
    """Sum of |term| of each output of ba_linearize: the stored rows (m,12) / (m,6) and rs (m,2) scaled by sqrt(rho'),
    Hcc (C,21), Hpp (P,6), gc (C,6), gp (P,3) and the cost."""
    r = ba_residual(poses, points, pix, cidx, pidx)
    Jc_abs, Jp_abs, rabs = ba_terms(poses, points, pix, cidx, pidx)
    rho, w = robust(kind, delta, (r ** 2).sum(-1))
    ww = w * _weight_factor(kind, delta, rabs)
    sw = np.sqrt(ww)
    C, P = poses.shape[0], points.shape[0]
    iu, iu3 = np.triu_indices(6), np.triu_indices(3)
    Hcc = _group_sum(cidx, np.einsum('mka,mkb->mab', Jc_abs, Jc_abs)[:, iu[0], iu[1]] * ww[:, None], C)
    Hpp = _group_sum(pidx, np.einsum('mka,mkb->mab', Jp_abs, Jp_abs)[:, iu3[0], iu3[1]] * ww[:, None], P)
    gc = _group_sum(cidx, np.einsum('mka,mk->ma', Jc_abs, rabs) * ww[:, None], C)
    gp = _group_sum(pidx, np.einsum('mka,mk->ma', Jp_abs, rabs) * ww[:, None], P)
    cost = _rho_terms(kind, delta, (r ** 2).sum(-1)).sum() + (w * 2 * (np.abs(r) * rabs).sum(-1)).sum()
    return ((Jc_abs * sw[:, None, None]).reshape(-1, 12), (Jp_abs * sw[:, None, None]).reshape(-1, 6), rabs * sw[:, None],
            Hcc, Hpp, gc, gp, np.array([cost]))


def ba_rows_from_y(y, sw, poses, cidx, absolute=False):
    """Stored BA rows rebuilt from the camera-frame point y and sqrt(rho') (the Y4 layout): Jc (m,2,6), Jp (m,2,3);
    with absolute=True their magnitudes (y taken as exact)."""
    m = len(y)
    z = y[:, 2]
    dpi = np.zeros((m, 2, 3))
    dpi[:, 0, 0] = dpi[:, 1, 1] = -1 / z
    dpi[:, 0, 2], dpi[:, 1, 2] = y[:, 0] / z ** 2, y[:, 1] / z ** 2
    dy = np.concatenate([np.broadcast_to(np.eye(3), (m, 3, 3)), O.vec2skew(-y)], -1)
    R = _rot(poses[cidx][:, 3:])
    if absolute:
        dpi, dy, R = np.abs(dpi), np.abs(dy), np.abs(R)
    s = np.abs(sw) if absolute else sw
    return dpi @ dy * s[:, None, None], dpi @ R * s[:, None, None]


# ------------------------------------------------------------------ predicted reductions x^T H x + 2 x^T g for any x
def pgo_predicted(M21, u, ei, ej, x, terms=False):
    """x^T H x + 2 x^T g of the pose graph from per-edge blocks: H = sum_e (e_i - e_j) M_e (e_i - e_j)^T, g = pgo_scatter's.
    terms=True: (value, sum of |term|)."""
    M = _triu_unpack(M21)
    d = x[ei] - x[ej]
    val = np.einsum('ea,eab,eb->', d, M, d) - 2 * (d * u).sum()
    if not terms:
        return val
    da = np.abs(x[ei]) + np.abs(x[ej])
    return val, np.einsum('ea,eab,eb->', da, np.abs(M), da) + 2 * (da * np.abs(u)).sum()


def ba_predicted(Jc, Jp, rs, cidx, pidx, xc, xp, terms=False):
    """sum_k (J_k x)^T (2 r_k + J_k x), J_k x = Jc_k xc[c_k] + Jp_k xp[p_k] (stored rows, (m,12) / (m,6)).
    terms=True: (value, sum of |term|)."""
    Jc, Jp = Jc.reshape(-1, 2, 6), Jp.reshape(-1, 2, 3)
    Jd = (Jc @ xc[cidx][..., None] + Jp @ xp[pidx][..., None])[..., 0]
    val = (Jd * (2 * rs + Jd)).sum()
    if not terms:
        return val
    Ja = (np.abs(Jc) @ np.abs(xc[cidx])[..., None] + np.abs(Jp) @ np.abs(xp[pidx])[..., None])[..., 0]
    return val, (Ja * (2 * np.abs(rs) + Ja)).sum()


def node_layout(ei, ej, N):
    """Node-ordered slots of the edges: edge e owns slot epos_i[e] in node ei[e]'s list and epos_j[e] in ej[e]'s; node n's
    slots are nptr[n] .. nptr[n+1], in the order of a stable sort of the keys [ei, ej]; nother[s] is the other endpoint."""
    ei, ej = np.asarray(ei, np.int64), np.asarray(ej, np.int64)
    E = len(ei)
    keys = np.concatenate([ei, ej])
    order = np.argsort(keys, kind="stable")
    pos = np.empty(2 * E, np.int64)
    pos[order] = np.arange(2 * E)
    nptr = np.concatenate([[0], np.cumsum(np.bincount(keys, minlength=N))])
    nother = np.concatenate([ej, ei])[order]
    return pos[:E], pos[E:], nptr, nother
