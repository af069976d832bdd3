"""fp64 numpy restatement of the BAL bundle-adjustment route (csrc/bal_math.cuh, csrc/bal.cu, optim/structured.py
BALProblem) and of the reference's dense LM on the same model (pypose/optim/optimizer.py:645-680).

    y = T_c p_j,   n = -y[:2] / y[2],   rho = |n|^2,   d = 1 + k1 rho + k2 rho^2,   r = f d n - z

Camera unknowns [xi (6, left SE3 perturbation) | f, k1, k2], point unknowns dp (3).  Test infrastructure only.
"""
import numpy as np

from oracle import lie_oracle as L


def problem(seed, C=8, P=60, M=400, scale=1.0, noise=0.5):
    """A seeded BAL-like problem: true parameters, noisy observations and a start perturbed by `scale` times
    (0.02 rad, 0.1 units, 1 % focal length, 0.01 k1, 0.001 k2, 0.05 units per point); pixel noise `noise`."""
    rng = np.random.default_rng(seed)
    T = L.exp("SE3", np.concatenate([rng.normal(0, 0.3, (C, 3)), rng.normal(0, 0.05, (C, 3))], 1))
    T[:, :3] = rng.normal(0, 0.3, (C, 3))
    # points 3-8 units in front of camera 0 (looking down -z), expressed in the world frame
    pc = np.concatenate([rng.uniform(-1.5, 1.5, (P, 2)), -rng.uniform(3.0, 8.0, (P, 1))], 1)
    pw = L.act("SE3", L.inv("SE3", T[:1].repeat(P, 0)), pc)
    K = np.stack([rng.uniform(450, 550, C), rng.uniform(-0.1, 0.1, C), rng.uniform(-0.01, 0.01, C)], 1)
    # every point seen by two different cameras, the rest of the observations at random
    c2 = np.stack([rng.permutation(C)[:2] for _ in range(P)])
    cidx = np.concatenate([c2[:, 0], c2[:, 1], rng.integers(0, C, M - 2 * P)])
    pidx = np.concatenate([np.arange(P), np.arange(P), rng.integers(0, P, M - 2 * P)])
    order = rng.permutation(M)
    cidx, pidx = cidx[order].astype(np.int64), pidx[order].astype(np.int64)
    pix = residual(K, T, pw, np.zeros((M, 2)), cidx, pidx) + rng.normal(0, noise, (M, 2))
    g, s = np.random.default_rng(100 + seed), scale
    T0 = L.mul("SE3", L.exp("SE3", np.concatenate([g.normal(0, 0.02 * s, (C, 3)), g.normal(0, 0.005 * s, (C, 3))], 1)), T)
    P0 = pw + g.normal(0, 0.05 * s, pw.shape)
    K0 = K * np.array([1.0 + 0.01 * s, 1.0, 1.0]) + np.stack([np.zeros(C), g.normal(0, 0.01 * s, C),
                                                               g.normal(0, 0.001 * s, C)], 1)
    return dict(K0=K0, T0=T0, P0=P0, pix=pix, cidx=cidx, pidx=pidx, K=K, T=T, Pw=pw)


def residual(K, T, pts, pix, cidx, pidx):
    y = L.act("SE3", T[cidx], pts[pidx])
    n = -y[:, :2] / y[:, 2:]
    rho = (n * n).sum(1, keepdims=True)
    k = K[cidx]
    return k[:, :1] * (1 + k[:, 1:2] * rho + k[:, 2:3] * rho ** 2) * n - pix


def rows(K, T, pts, cidx, pidx):
    """Analytic Jacobian rows: Jc (M,2,9) = d r / d [xi | f, k1, k2], Jp (M,2,3) = d r / d p."""
    y = L.act("SE3", T[cidx], pts[pidx])
    k = K[cidx]
    f, k1, k2 = k[:, 0], k[:, 1], k[:, 2]
    n = -y[:, :2] / y[:, 2:]
    rho = (n * n).sum(1)
    d = 1 + k1 * rho + k2 * rho ** 2
    e = 2 * (k1 + 2 * k2 * rho)
    A = f[:, None, None] * (d[:, None, None] * np.eye(2) + e[:, None, None] * n[:, :, None] * n[:, None, :])
    z = y[:, 2]
    B = np.zeros((len(y), 2, 3))
    B[:, 0, 0] = B[:, 1, 1] = -1 / z
    B[:, 0, 2], B[:, 1, 2] = y[:, 0] / z ** 2, y[:, 1] / z ** 2
    G = A @ B                                                        # d r / d y
    Dxi = np.concatenate([np.broadcast_to(np.eye(3), (len(y), 3, 3)), -skew(y)], 2)
    R = quat_to_mat(T[cidx, 3:])
    Jc = np.concatenate([G @ Dxi, (d[:, None] * n)[:, :, None], (f * rho)[:, None, None] * n[:, :, None],
                         (f * rho ** 2)[:, None, None] * n[:, :, None]], 2)
    Jp = G @ R
    return Jc, Jp


def skew(v):
    S = np.zeros(v.shape[:-1] + (3, 3))
    S[..., 0, 1], S[..., 0, 2], S[..., 1, 2] = -v[..., 2], v[..., 1], -v[..., 0]
    return S - np.swapaxes(S, -1, -2)


def quat_to_mat(q):
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def robust(kind, delta, x):
    """rho(x) and rho'(x) on x = |r|^2 for kind 0 (none), 1 (Huber), 3 (Cauchy) (optim/kernel.py)."""
    if kind == 1:
        root = np.sqrt(x)
        inside = root < delta
        return np.where(inside, x, 2 * delta * root - delta ** 2), np.where(inside, 1.0, delta / root)
    if kind == 3:
        q = x / delta ** 2 + 1
        return delta ** 2 * np.log(q), 1 / q
    return x, np.ones_like(x)


def blocks(K, T, pts, pix, cidx, pidx, kind=0, delta=1.0):
    """FastTriggs-scaled rows and the block sums: Hcc (C,9,9), gc (C,9), Hpp (P,3,3), gp (P,3), loss, Jc, Jp, r."""
    r = residual(K, T, pts, pix, cidx, pidx)
    rho, w = robust(kind, delta, (r * r).sum(1))
    sw = np.sqrt(w) if kind else np.ones_like(w)
    Jc, Jp = rows(K, T, pts, cidx, pidx)
    Jc, Jp, rs = Jc * sw[:, None, None], Jp * sw[:, None, None], r * sw[:, None]
    C, P = len(K), len(pts)
    Hcc, gc = np.zeros((C, 9, 9)), np.zeros((C, 9))
    Hpp, gp = np.zeros((P, 3, 3)), np.zeros((P, 3))
    np.add.at(Hcc, cidx, np.swapaxes(Jc, 1, 2) @ Jc)
    np.add.at(gc, cidx, np.einsum("kia,ki->ka", Jc, rs))
    np.add.at(Hpp, pidx, np.swapaxes(Jp, 1, 2) @ Jp)
    np.add.at(gp, pidx, np.einsum("kia,ki->ka", Jp, rs))
    return dict(Hcc=Hcc, gc=gc, Hpp=Hpp, gp=gp, loss=rho.sum(), Jc=Jc, Jp=Jp, rs=rs)


def damp(H, scale, dmin, dmax):
    H = H.copy()
    i = np.arange(H.shape[-1])
    H[..., i, i] = np.clip(H[..., i, i], dmin, dmax) * scale
    return H


def wv(Jc, Jp, cidx, pidx, t, C):
    """W t: y[c] = sum_k Jc_k^T Jp_k t[j_k]  (C,9)."""
    y = np.zeros((C, 9))
    np.add.at(y, cidx, np.einsum("kia,kib,kb->ka", Jc, Jp, t[pidx]))
    return y


def wtx(Jc, Jp, cidx, pidx, x, P):
    """W^T x: u[j] = sum_k Jp_k^T Jc_k x[c_k]  (P,3)."""
    u = np.zeros((P, 3))
    np.add.at(u, pidx, np.einsum("kia,kib,kb->ka", Jp, Jc, x[cidx]))
    return u


def schur(b, cidx, pidx, scale, dmin=1e-6, dmax=1e32):
    """Damped reduced camera system S dc = rhs with its diagonal blocks Sd: returns S (9C,9C), rhs (9C), Sd (C,9,9),
    Hpinv (P,3,3)."""
    C, P = len(b["gc"]), len(b["gp"])
    Hc, Hpinv = damp(b["Hcc"], scale, dmin, dmax), np.linalg.inv(damp(b["Hpp"], scale, dmin, dmax))
    Jc, Jp = b["Jc"], b["Jp"]
    Wk = np.swapaxes(Jc, 1, 2) @ Jp                                    # (M,9,3)
    W = np.zeros((9 * C, 3 * P))
    for k in range(len(cidx)):
        W[9 * cidx[k]:9 * cidx[k] + 9, 3 * pidx[k]:3 * pidx[k] + 3] += Wk[k]
    Hpi = np.zeros((3 * P, 3 * P))
    for j in range(P):
        Hpi[3 * j:3 * j + 3, 3 * j:3 * j + 3] = Hpinv[j]
    Hcd = np.zeros((9 * C, 9 * C))
    for c in range(C):
        Hcd[9 * c:9 * c + 9, 9 * c:9 * c + 9] = Hc[c]
    S = Hcd - W @ Hpi @ W.T
    rhs = -b["gc"].reshape(-1) + W @ Hpi @ b["gp"].reshape(-1)
    Sd = np.stack([S[9 * c:9 * c + 9, 9 * c:9 * c + 9] for c in range(C)])
    return S, rhs, Sd, Hpinv


def dense_step(b, cidx, pidx, scale, dmin=1e-6, dmax=1e32):
    """The damped LM step over all unknowns by a dense solve: (xc (C,9), xp (P,3)), and its predicted reduction."""
    S, rhs, _, Hpinv = schur(b, cidx, pidx, scale, dmin, dmax)
    xc = np.linalg.solve(S, rhs).reshape(-1, 9)
    xp = -np.einsum("jab,jb->ja", Hpinv, b["gp"] + wtx(b["Jc"], b["Jp"], cidx, pidx, xc, len(b["gp"])))
    Jd = np.einsum("kia,ka->ki", b["Jc"], xc[cidx]) + np.einsum("kia,ka->ki", b["Jp"], xp[pidx])
    return xc, xp, float((Jd * (2 * b["rs"] + Jd)).sum())


def retract(K, T, pts, xc, xp):
    return K + xc[:, 6:], L.mul("SE3", L.exp("SE3", xc[:, :6]), T), pts + xp


def lm(K, T, pts, pix, cidx, pidx, steps, strategy="constant", damping=1e-6, reject=16, dmin=1e-6, dmax=1e32):
    """The reference's dense LM (optimizer.py:659-680) with Constant(damping) or TrustRegion() (strategy.py) in fp64."""
    tr = dict(radius=1e6, damping=1e-6, down=0.5)               # TrustRegion() defaults
    dmp = tr["damping"] if strategy == "trustregion" else damping
    loss_h, Ks, Ts, Ps, rej = [], [], [], [], []
    last = None
    for _ in range(steps):
        b = blocks(K, T, pts, pix, cidx, pidx)
        cur = b["loss"] if last is None else last
        scale, nrej = 1.0, 0
        while True:
            scale *= 1 + dmp
            xc, xp, pred = dense_step(b, cidx, pidx, scale, dmin, dmax)
            Kt, Tt, Pt = retract(K, T, pts, xc, xp)
            loss = blocks(Kt, Tt, Pt, pix, cidx, pidx)["loss"]
            if strategy == "trustregion":                       # strategy.py TrustRegion.update
                quality = (cur - loss) / -pred
                radius = 1.0 / dmp
                if quality > 0.5:
                    radius, tr["down"] = 2.0 * radius, 0.5
                elif quality > 1e-3:
                    tr["down"] = 0.5
                else:
                    radius, tr["down"] = radius * tr["down"], tr["down"] * 0.5
                tr["down"] = max(1e-6, min(tr["down"], 1e16))
                dmp = 1.0 / max(1e-6, min(radius, 1e16))
            if cur < loss and nrej < reject:
                nrej += 1
                continue
            K, T, pts, last = Kt, Tt, Pt, loss
            break
        loss_h.append(last); Ks.append(K); Ts.append(T); Ps.append(pts); rej.append(nrej)
    return dict(loss=np.array(loss_h), K=np.stack(Ks), T=np.stack(Ts), P=np.stack(Ps), reject=np.array(rej))
