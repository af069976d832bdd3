"""CPU oracle for the LieTensor op family — TEST INFRASTRUCTURE ONLY.

A numpy restatement of the reference algorithm (pypose v0.9.5, pypose/lietensor/operation.py and
lietensor.py; cited per function as op.py:LINE / lt.py:LINE), written in the reference's own
*matrix* form (explicit 3x3 / 6x6 / 7x7 Jacobians and `g @ J` products) so that it is an
independent derivation from the cross-product forms used by the CUDA kernels.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
The shipped package (pypose_b200/) never does: it has no CPU path at all.

Parity of this oracle is pinned by tests/test_oracle_golden.py against tests/golden/*.npz, which
were produced by importing the reference itself (oracle/make_golden.py, run against the
reference checkout named by PYPOSE_REFERENCE).

Entry point: run(symbol, *arrays) with the same names / argument order as the C-ABI
(include/b200pose.h) minus the `b200_` prefix and dtype suffix, e.g. run("SE3_log_bwd", x, g).
"""
import numpy as np

GROUPS = {"SO3": ("so3", 4, 3), "SE3": ("se3", 7, 6), "RxSO3": ("rxso3", 5, 4), "Sim3": ("sim3", 8, 7)}
ALG2GRP = {v[0]: k for k, v in GROUPS.items()}


# Reference behaviour: Taylor branches only when theta <= eps (op.py:12, 27, 43).  In fp64 the closed forms
# lose up to ~1e-4 absolute accuracy for theta in (eps, 1e-3] (SURVEY.md §8c).  `wide_taylor()` switches the
# SAME formulas to their Taylor series over theta < 1e-2 (with two more terms) — used only by the tiny-angle
# parity rows, where "the reference evaluated exactly" is the truth rather than its rounding noise.
_WIDE = [False]


class wide_taylor:
    def __enter__(self):
        _WIDE[0] = True

    def __exit__(self, *a):
        _WIDE[0] = False


def _eps(x):
    return 1e-2 if _WIDE[0] else np.finfo(x.dtype).eps


def _hi(th2, c4, c6):
    """extra Taylor terms (theta^4, theta^6) enabled in wide mode only."""
    return (c4 * th2 * th2 + c6 * th2 * th2 * th2) if _WIDE[0] else 0.0


def pm(x):
    """basics/ops.py:26 — sign with pm(0) = +1."""
    return np.sign(np.sign(x) * 2 + 1)


def vec2skew(v):
    """lietensor/basics.py:36-41."""
    O = np.zeros(v.shape[:-1], dtype=v.dtype)
    return np.stack([np.stack([O, -v[..., 2], v[..., 1]], -1),
                     np.stack([v[..., 2], O, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], O], -1)], -2)


def _eye(n, like, batch):
    return np.broadcast_to(np.eye(n, dtype=like.dtype), batch + (n, n)).copy()


def _where(cond, a_fn, b_fn):
    with np.errstate(all="ignore"):
        return np.where(cond, np.nan_to_num(a_fn()), np.nan_to_num(b_fn()))


# ------------------------------------------------------------------ Jacobian helpers
def so3_Jl(x):
    """op.py:7-20."""
    K = vec2skew(x)
    th = np.linalg.norm(x, axis=-1)[..., None, None]
    th2 = th * th
    big = th > _eps(x)
    c1 = _where(big, lambda: (1 - np.cos(th)) / th2, lambda: 0.5 - th2 / 24.0 + _hi(th2, 1 / 720, -1 / 40320))
    c2 = _where(big, lambda: (th - np.sin(th)) / (th * th2),
                lambda: 1.0 / 6 - th2 / 120.0 + _hi(th2, 1 / 5040, -1 / 362880))
    return _eye(3, x, x.shape[:-1]) + c1 * K + c2 * (K @ K)


def so3_Jl_inv(x):
    """op.py:23-32."""
    K = vec2skew(x)
    th = np.linalg.norm(x, axis=-1)[..., None, None]
    big = th > _eps(x)
    c = _where(big, lambda: (1.0 - th * np.cos(0.5 * th) / (2.0 * np.sin(0.5 * th))) / (th * th),
               lambda: np.full_like(th, 1.0 / 12) + ((th * th / 720 + _hi(th * th, 1 / 30240, 1 / 1209600)) if _WIDE[0] else 0.0))
    return _eye(3, x, x.shape[:-1]) - 0.5 * K + c * (K @ K)


def calcQ(x):
    """op.py:37-58."""
    tau, phi = x[..., :3], x[..., 3:]
    T, P = vec2skew(tau), vec2skew(phi)
    th = np.linalg.norm(phi, axis=-1)[..., None, None]
    th2 = th * th
    th4 = th2 * th2
    big = th > _eps(x)
    c1 = _where(big, lambda: (th - np.sin(th)) / (th2 * th), lambda: 1.0 / 6 - th2 / 120.0 + _hi(th2, 1 / 5040, -1 / 362880))
    c2 = _where(big, lambda: (th2 + 2 * np.cos(th) - 2) / (2 * th4),
                lambda: 1.0 / 24 - th2 / 720.0 + _hi(th2, 1 / 40320, -1 / 3628800))
    c3 = _where(big, lambda: (2 * th - 3 * np.sin(th) + th * np.cos(th)) / (2 * th4 * th),
                lambda: 1.0 / 120 - th2 / 2520.0 + _hi(th2, 1 / 120960, -1 / 9979200))
    return (0.5 * T + c1 * (P @ T + T @ P + P @ T @ P)
            + c2 * (P @ P @ T + T @ P @ P - 3 * P @ T @ P) + c3 * (P @ T @ P @ P + P @ P @ T @ P))


def _block(rows):
    return np.concatenate([np.concatenate(r, -1) for r in rows], -2)


def se3_Jl(x):
    """op.py:61-65."""
    J = so3_Jl(x[..., 3:])
    Z = np.zeros_like(J)
    return _block([[J, calcQ(x)], [Z, J]])


def se3_Jl_inv(x):
    """op.py:68-75."""
    Ji, Q = so3_Jl_inv(x[..., 3:]), calcQ(x)
    Z = np.zeros_like(Ji)
    return _block([[Ji, -Ji @ Q @ Ji], [Z, Ji]])


def so3_adj(x):
    return vec2skew(x)


def se3_adj(x):
    """op.py:77-83."""
    P, T = vec2skew(x[..., 3:]), vec2skew(x[..., :3])
    return _block([[P, T], [np.zeros_like(P), P]])


def rxso3_Ws(x):
    """op.py:85-129 (four (sigma, theta) cases)."""
    rot, sigma = x[..., :3], x[..., 3]
    th = np.linalg.norm(rot, axis=-1)
    sl, tl = np.abs(sigma) > np.finfo(x.dtype).eps, th > np.finfo(x.dtype).eps
    s, s2, t2 = np.exp(sigma), sigma * sigma, th * th
    with np.errstate(all="ignore"):
        C = np.where(sl, (np.expm1(sigma) if _WIDE[0] else (s - 1.0)) / sigma, 1.0)   # wide: no (e^s - 1) cancellation
        A1, B1 = 0.5, 1.0 / 6
        A2, B2 = (1.0 - np.cos(th)) / t2, (th - np.sin(th)) / (t2 * th)
        if _WIDE[0]:
            sm = th < 1e-2
            A2 = np.where(sm, 0.5 - t2 / 24 + t2 * t2 / 720, A2)
            B2 = np.where(sm, 1.0 / 6 - t2 / 120 + t2 * t2 / 5040, B2)
        A3 = (1.0 + (sigma - 1.0) * s) / s2
        B3 = (0.5 * s2 * s + s - 1.0 - s2 * s) / (s2 * sigma)   # as written in the reference (op.py:112)
        a, b, c = s * np.sin(th), s * np.cos(th), t2 + s2
        A4 = (a * sigma + (1 - b) * th) / (th * c)
        B4 = (C - ((b - 1) * sigma + a * th) / c) / t2
        A = np.where(~sl & ~tl, A1, np.where(~sl & tl, A2, np.where(sl & ~tl, A3, A4)))
        B = np.where(~sl & ~tl, B1, np.where(~sl & tl, B2, np.where(sl & ~tl, B3, B4)))
    K = vec2skew(rot)
    A, B, C = (np.nan_to_num(v)[..., None, None] for v in (A, B, C))
    return A * K + B * (K @ K) + C * _eye(3, x, x.shape[:-1])


def rxso3_Jl(x):
    """op.py:132-135."""
    J = _eye(4, x, x.shape[:-1])
    J[..., :3, :3] = so3_Jl(x[..., :3])
    return J


def rxso3_Jl_inv(x):
    """op.py:137-140."""
    J = _eye(4, x, x.shape[:-1])
    J[..., :3, :3] = so3_Jl_inv(x[..., :3])
    return J


def rxso3_adj(x):
    """op.py:142-145."""
    ad = np.zeros(x.shape[:-1] + (4, 4), dtype=x.dtype)
    ad[..., :3, :3] = vec2skew(x[..., :3])
    return ad


def sim3_adj(x):
    """op.py:147-156."""
    tau, phi, sigma = x[..., :3], x[..., 3:6], x[..., 6:]
    ad = np.zeros(x.shape[:-1] + (7, 7), dtype=x.dtype)
    ad[..., :3, :3] = vec2skew(phi) + sigma[..., None] * np.eye(3, dtype=x.dtype)
    ad[..., :3, 3:6] = vec2skew(tau)
    ad[..., :3, 6] = -tau
    ad[..., 3:6, 3:6] = vec2skew(phi)
    return ad


def sim3_Jl(x):
    """op.py:159-164 (truncated series, approximate by design)."""
    Xi = sim3_adj(x)
    Xi2 = Xi @ Xi
    Xi4 = Xi2 @ Xi2
    I = _eye(7, x, x.shape[:-1])
    return I + Xi / 2 + Xi2 / 6 + (Xi @ Xi2) / 24 + Xi4 / 120 + (Xi @ Xi4) / 720


def sim3_Jl_inv(x):
    """op.py:167-172."""
    Xi = sim3_adj(x)
    Xi2 = Xi @ Xi
    Xi4 = Xi2 @ Xi2
    return _eye(7, x, x.shape[:-1]) - Xi / 2 + Xi2 / 12 - Xi4 / 720


def SO3_Adj(X):
    """op.py:175-179 (rotation matrix of a quaternion)."""
    I = np.eye(3, dtype=X.dtype)
    v, w = X[..., :3], X[..., 3:]
    return 2.0 * w[..., None] * (w[..., None] * I + vec2skew(v)) - I + 2.0 * v[..., :, None] * v[..., None, :]


def SE3_Adj(X):
    """op.py:202-210."""
    R = SO3_Adj(X[..., 3:])
    return _block([[R, vec2skew(X[..., :3]) @ R], [np.zeros_like(R), R]])


def RxSO3_Adj(X):
    """op.py:237-240."""
    A = _eye(4, X, X.shape[:-1])
    A[..., :3, :3] = SO3_Adj(X[..., :4])
    return A


def Sim3_Adj(X):
    """op.py:268-276."""
    A = _eye(7, X, X.shape[:-1])
    R = SO3_Adj(X[..., 3:7])
    A[..., :3, :3] = X[..., 7:, None] * R
    A[..., :3, 3:6] = vec2skew(X[..., :3]) @ R
    A[..., :3, 6] = -X[..., :3]
    A[..., 3:6, 3:6] = R
    return A


JL = {"SO3": so3_Jl, "SE3": se3_Jl, "RxSO3": rxso3_Jl, "Sim3": sim3_Jl}
JLINV = {"SO3": so3_Jl_inv, "SE3": se3_Jl_inv, "RxSO3": rxso3_Jl_inv, "Sim3": sim3_Jl_inv}
LITTLE_AD = {"SO3": so3_adj, "SE3": se3_adj, "RxSO3": rxso3_adj, "Sim3": sim3_adj}
ADJ = {"SO3": SO3_Adj, "SE3": SE3_Adj, "RxSO3": RxSO3_Adj, "Sim3": Sim3_Adj}


def _rowmat(g, M):
    """g @ M for row vectors."""
    return (g[..., None, :] @ M)[..., 0, :]


def _matvec(M, v):
    return (M @ v[..., :, None])[..., 0]


def _pad0(g):
    return np.concatenate([g, np.zeros(g.shape[:-1] + (1,), dtype=g.dtype)], -1)


# ------------------------------------------------------------------ forward ops
def so3_exp(x):
    """op.py:343-357."""
    th = np.linalg.norm(x, axis=-1, keepdims=True)
    th2 = th * th
    th4 = th2 * th2
    big = th > np.finfo(x.dtype).eps
    im = _where(big, lambda: np.sin(0.5 * th) / th, lambda: 0.5 - th2 / 48.0 + th4 / 3840.0)
    re = _where(big, lambda: np.cos(0.5 * th), lambda: 1.0 - th2 / 8.0 + th4 / 384.0)
    return np.concatenate([x * im, re], -1)


def SO3_log(X):
    """op.py:308-324."""
    eps = np.finfo(X.dtype).eps
    v, w = X[..., :3], X[..., 3:]
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    vl, wl = n > eps, np.abs(w) > eps
    with np.errstate(all="ignore"):
        f1 = np.nan_to_num(2.0 * np.arctan(n / w) / n)
        f2 = np.nan_to_num(pm(w) * np.pi / n)
        f3 = np.nan_to_num(2.0 * (1.0 / w - n * n / (3 * w ** 3)))
    factor = (vl & wl) * f1 + (vl & ~wl) * f2 + (~vl) * f3
    return factor * v


def SO3_act(X, p):
    """op.py:520-525."""
    v, w = X[..., :3], X[..., 3:]
    uv = np.cross(v, p)
    uv = uv + uv
    return p + w * uv + np.cross(v, uv)


def SO3_mul(X, Y):
    """op.py:833-837."""
    xv, xw, yv, yw = X[..., :3], X[..., 3:], Y[..., :3], Y[..., 3:]
    zv = xw * yv + xv * yw + np.cross(xv, yv)
    zw = xw * yw - (xv * yv).sum(-1, keepdims=True)
    return np.concatenate([zv, zw], -1)


def SO3_inv(X):
    return np.concatenate([-X[..., :3], X[..., 3:]], -1)


def exp(grp, x):
    if grp == "SO3":
        return so3_exp(x)
    if grp == "SE3":      # op.py:401-405
        t = _matvec(so3_Jl(x[..., 3:]), x[..., :3])
        return np.concatenate([t, so3_exp(x[..., 3:])], -1)
    if grp == "RxSO3":    # op.py:448-451
        return np.concatenate([so3_exp(x[..., :3]), np.exp(x[..., 3:])], -1)
    # Sim3: op.py:496-500
    t = _matvec(rxso3_Ws(x[..., 3:]), x[..., :3])
    return np.concatenate([t, so3_exp(x[..., 3:6]), np.exp(x[..., 6:])], -1)


def log(grp, X):
    if grp == "SO3":
        return SO3_log(X)
    if grp == "SE3":      # op.py:377-382
        phi = SO3_log(X[..., 3:])
        return np.concatenate([_matvec(so3_Jl_inv(phi), X[..., :3]), phi], -1)
    if grp == "RxSO3":    # op.py:425-428
        return np.concatenate([SO3_log(X[..., :4]), np.log(X[..., 4:])], -1)
    ps = np.concatenate([SO3_log(X[..., 3:7]), np.log(X[..., 7:])], -1)   # op.py:471-476
    tau = _matvec(np.linalg.inv(rxso3_Ws(ps)), X[..., :3])
    return np.concatenate([tau, ps], -1)


def _split(grp, X):
    """-> (t or None, q, s or None)"""
    if grp == "SO3":
        return None, X, None
    if grp == "SE3":
        return X[..., :3], X[..., 3:], None
    if grp == "RxSO3":
        return None, X[..., :4], X[..., 4:]
    return X[..., :3], X[..., 3:7], X[..., 7:]


def _join(grp, t, q, s):
    parts = ([t] if t is not None else []) + [q] + ([s] if s is not None else [])
    return np.concatenate(parts, -1)


def act(grp, X, p):
    """op.py:516-603."""
    t, q, s = _split(grp, X)
    o = SO3_act(q, p)
    if s is not None:
        o = s * o
    if t is not None:
        o = t + o
    return o


def act4(grp, X, p):
    """op.py:623-706."""
    t, q, s = _split(grp, X)
    o = SO3_act(q, p[..., :3])
    if s is not None:
        o = s * o
    if t is not None:
        o = o + t * p[..., 3:]
    return np.concatenate([o, p[..., 3:]], -1)


def inv(grp, X):
    """op.py:930-1008."""
    t, q, s = _split(grp, X)
    qi = SO3_inv(q)
    si = None if s is None else 1.0 / s
    ti = None
    if t is not None:
        r = SO3_act(qi, t)
        ti = -(r if si is None else si * r)
    return _join(grp, ti, qi, si)


def mul(grp, X, Y):
    """op.py:829-912."""
    tx, qx, sx = _split(grp, X)
    ty, qy, sy = _split(grp, Y)
    q = SO3_mul(qx, qy)
    s = None if sx is None else sx * sy
    t = None
    if tx is not None:
        r = SO3_act(qx, ty)
        t = tx + (r if sx is None else sx * r)
    return _join(grp, t, q, s)


def adj(grp, X, a):
    """op.py:725-810: Adj(X) a."""
    return _matvec(ADJ[grp](X), a)


def adjt(grp, X, a):
    """op.py:1024-1099: Adj(X^-1) a."""
    return adj(grp, inv(grp, X), a)


def jinvp(grp, X, p):
    """lt.py:257-264, 422-429, 556-563, 700-707."""
    return _matvec(JLINV[grp](log(grp, X)), p)


def so3_jr(x):
    """lt.py:343-351."""
    K = vec2skew(x)
    th = np.linalg.norm(x, axis=-1)[..., None, None]
    I = _eye(3, x, x.shape[:-1])
    with np.errstate(all="ignore"):
        Jr = I - (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * (K @ K)
    if _WIDE[0]:
        t2 = th * th
        Js = I - (0.5 - t2 / 24 + t2 * t2 / 720) * K + (1.0 / 6 - t2 / 120 + t2 * t2 / 5040) * (K @ K)
        return np.where(th > 1e-2, Jr, Js)
    return np.where(th > np.finfo(x.dtype).eps, Jr, I)


# ------------------------------------------------------------------ backward rules
def exp_bwd(grp, x, gX):
    K = GROUPS[grp][2]
    return _rowmat(gX[..., :K], JL[grp](x))


def log_bwd(grp, out, g):
    return _pad0(_rowmat(g, JLINV[grp](out)))


def inv_bwd(grp, Y, gY):
    K = GROUPS[grp][2]
    return _pad0(-_rowmat(gY[..., :K], ADJ[grp](Y)))


def mul_bwd(grp, X, gZ):
    K = GROUPS[grp][2]
    g = gZ[..., :K]
    return _pad0(g), _pad0(_rowmat(g, ADJ[grp](X)))


def _act_jac(grp, o):
    """op.py:186-301 *_Act_Jacobian."""
    I = np.broadcast_to(np.eye(3, dtype=o.dtype), o.shape[:-1] + (3, 3))
    S = vec2skew(-o)
    if grp == "SO3":
        return S
    if grp == "SE3":
        return np.concatenate([I, S], -1)
    if grp == "RxSO3":
        return np.concatenate([S, o[..., :, None]], -1)
    return np.concatenate([I, S, o[..., :, None]], -1)


def _matrix3(grp, X):
    _, q, s = _split(grp, X)
    R = SO3_Adj(q)
    return R if s is None else s[..., None] * R


def act_bwd(grp, X, out, g):
    return _pad0(_rowmat(g, _act_jac(grp, out))), _rowmat(g, _matrix3(grp, X))


def _act4_jac(grp, p):
    K = GROUPS[grp][2]
    J = np.zeros(p.shape[:-1] + (4, K), dtype=p.dtype)
    S = vec2skew(-p[..., :3])
    I = np.eye(3, dtype=p.dtype)
    if grp == "SO3":
        J[..., :3, :3] = S
    elif grp == "SE3":
        J[..., :3, :3] = I * p[..., 3:, None]
        J[..., :3, 3:] = S
    elif grp == "RxSO3":
        J[..., :3, :3] = S
        J[..., :3, 3] = p[..., :3]
    else:
        J[..., :3, :3] = I * p[..., 3:, None]
        J[..., :3, 3:6] = S
        J[..., :3, 6] = p[..., :3]
    return J


def _matrix4(grp, X):
    t, _, _ = _split(grp, X)
    M = _eye(4, X, X.shape[:-1])
    M[..., :3, :3] = _matrix3(grp, X)
    if t is not None:
        M[..., :3, 3] = t
    return M


def act4_bwd(grp, X, out, g):
    return _pad0(_rowmat(g, _act4_jac(grp, out))), _rowmat(g, _matrix4(grp, X))


def adj_bwd(grp, X, out, g):
    return _pad0(-_rowmat(g, LITTLE_AD[grp](out))), _rowmat(g, ADJ[grp](X))


def adjt_bwd(grp, X, a, g):
    ga = adj(grp, X, g)
    return _pad0(-_rowmat(a, LITTLE_AD[grp](ga))), ga


_FWD1 = {"exp_fwd": exp, "log_fwd": log, "inv_fwd": inv}
_FWD2 = {"mul_fwd": mul, "act_fwd": act, "act4_fwd": act4, "adj_fwd": adj, "adjt_fwd": adjt, "jinvp_fwd": jinvp}
_BWD = {"exp_bwd": exp_bwd, "log_bwd": log_bwd, "inv_bwd": inv_bwd, "mul_bwd": mul_bwd, "act_bwd": act_bwd,
        "act4_bwd": act4_bwd, "adj_bwd": adj_bwd, "adjt_bwd": adjt_bwd}


def run(symbol, *arrays):
    """Evaluate the oracle for C-ABI entry `b200_<symbol>_<dtype>`; returns a list of outputs."""
    if symbol == "so3_jr":
        J = so3_jr(arrays[0])
        return [J.reshape(J.shape[:-2] + (9,))]
    prefix, op = symbol.split("_", 1)
    grp = ALG2GRP.get(prefix, prefix)
    arrays = [np.asarray(a) for a in arrays]
    if op in _FWD1:
        out = _FWD1[op](grp, *arrays)
    elif op in _FWD2:
        out = _FWD2[op](grp, *arrays)
    else:
        out = _BWD[op](grp, *arrays)
    return list(out) if isinstance(out, tuple) else [out]
