"""fp64 numpy oracle of pp.knn, the Kabsch rule and pp.module.ICP with the ReduceToBason stop rule (DESIGN.md §3.4).

Test infrastructure only: the package never imports it.
"""
import numpy as np

KABSCH_EPS = {np.float32: 1e-6, np.float64: 1e-12}


def _norm(diff, ord):
    a = np.abs(diff)
    if ord == 2:
        return np.sqrt((diff * diff).sum(-1))
    if ord == 1:
        return a.sum(-1)
    return a.max(-1)


def distances(ref, nbr, ord=2):
    """(..., N1, D), (..., N2, D) -> (..., N1, N2) in fp64."""
    ref, nbr = np.asarray(ref, np.float64), np.asarray(nbr, np.float64)
    return _norm(ref[..., :, None, :] - nbr[..., None, :, :], ord)


def knn(ref, nbr, k=1, ord=2, largest=False):
    """Brute force; equal distances list the lower index first.  -> values (..., N1, k), indices (..., N1, k)."""
    d = distances(ref, nbr, ord)
    idx = np.argsort(-d if largest else d, axis=-1, kind="stable")[..., :k]
    return np.take_along_axis(d, idx, -1), idx


def kabsch(H, eps):
    """The rotation of the Kabsch step for the cross-covariance H (sum t s^T of the centred pairs)."""
    U, s, Vt = np.linalg.svd(np.asarray(H, np.float64))
    u, v = U.T.copy(), Vt.copy()                       # rows: singular vectors
    if not s[0] > 0:
        return np.eye(3)
    if s[1] <= eps * s[0]:                             # rank 1: smallest rotation v1 -> u1
        a, c = np.cross(v[0], u[0]), float(v[0] @ u[0])
        if 1.0 + c > 1e-12:
            K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
            return c * np.eye(3) + K + np.outer(a, a) / (1.0 + c)
        e = np.zeros(3)
        e[int(np.argmin(np.abs(v[0])))] = 1.0
        n = np.cross(v[0], e)
        n /= np.linalg.norm(n)
        return 2.0 * np.outer(n, n) - np.eye(3)
    if s[2] <= eps * s[0]:                             # rank 2: right-handed completion of both bases
        u[2], v[2] = np.cross(u[0], u[1]), np.cross(v[0], v[1])
        return u.T @ v
    R = u.T @ v
    if abs(np.linalg.det(R) + 1.0) < 1e-6:
        R = -R
    return R


def kabsch_cost(R, src, tgt):
    """sum |(t - mt) - R (s - ms)|^2 of associated point sets (N, 3)."""
    cs, ct = src - src.mean(0), tgt - tgt.mean(0)
    return float(((ct - cs @ R.T) ** 2).sum())


def quat2mat(q):
    x, y, z, w = q
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def se3_to_mat(T):
    """(..., 7) SE3 [t, q] -> (..., 3, 4)."""
    T = np.asarray(T, np.float64)
    out = np.zeros(T.shape[:-1] + (3, 4))
    for i in np.ndindex(T.shape[:-1]):
        out[i][:, :3] = quat2mat(T[i][3:])
        out[i][:, 3] = T[i][:3]
    return out


class ReduceToBason:
    """The stop rule evaluated in a given dtype (the loss dtype)."""

    def __init__(self, steps, patience=5, decreasing=1e-3, tol=1e-5, dtype=np.float64):
        self.max_steps, self.patience, self.decreasing, self.tol, self.dt = steps, patience, decreasing, tol, dtype
        self.steps, self.count, self.continual = 0, 0, True
        self.last = None

    def step(self, loss):
        dt = self.dt
        loss = np.atleast_1d(np.asarray(loss, dt))
        last = np.full_like(loss, np.inf) if self.last is None else self.last
        self.steps += 1
        if np.all(loss < dt(self.tol)):
            self.continual = False
        if self.steps >= self.max_steps:
            self.continual = False
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = ((last - loss).astype(dt) / loss).astype(dt)
        self.count = self.count + 1 if np.all(rel < dt(self.decreasing)) else 0
        self.last = loss
        if self.count >= self.patience:
            self.continual = False


def nearest(P, T, ord=2, matcher="brute", block=2048):
    """Nearest target of every point: P (Np, 3), T (Nt, 3) -> (distances (Np,), indices (Np,)) in fp64.

    "brute": exact, the first minimum (lower index) on ties, in query blocks of `block` rows, so memory stays at
    block * Nt * 3 values.  "kdtree": scipy's cKDTree, for clouds too large for brute force; the same distances, but an
    exact tie may pick either index, so use it on clouds whose nearest neighbours are unambiguous."""
    if matcher == "kdtree":
        from scipy.spatial import cKDTree
        d, j = cKDTree(T).query(P, k=1, p=np.inf if ord not in (1, 2) else ord)
        return d, j
    d, j = np.empty(len(P)), np.empty(len(P), np.int64)
    for i in range(0, len(P), block):
        dd, jj = knn(P[i:i + block], T, 1, ord)
        d[i:i + block], j[i:i + block] = dd[:, 0], jj[:, 0]
    return d, j


def icp(source, target, init=None, ord=2, steps=200, patience=5, decreasing=1e-3, tol=1e-5, eps=1e-12, matcher="brute",
        stepper=None):
    """Point-to-point ICP in fp64.  source (..., Ns, 3), target (..., Nt, 3), init (..., 4, 4)/(...,3,4) or None
    -> A (B, 3, 4) over the flattened broadcast batch, per-step losses (steps, B), batch shape.

    Matching runs per batch element (see `nearest` for `matcher`), so memory does not grow with the batch.  `stepper`
    replaces the ReduceToBason(steps, patience, decreasing, tol) stop rule (any object with `step(loss)` and `continual`)."""
    source, target = np.asarray(source, np.float64), np.asarray(target, np.float64)
    batch = np.broadcast_shapes(source.shape[:-2], target.shape[:-2], () if init is None else np.shape(init)[:-2])
    S = np.broadcast_to(source, batch + source.shape[-2:]).reshape(-1, *source.shape[-2:])
    Tg = np.broadcast_to(target, batch + target.shape[-2:]).reshape(-1, *target.shape[-2:])
    B = S.shape[0]
    A = np.tile(np.eye(4)[:3], (B, 1, 1))
    if init is not None:
        A = np.broadcast_to(np.asarray(init, np.float64)[..., :3, :], batch + (3, 4)).reshape(B, 3, 4).copy()
    st = ReduceToBason(steps, patience, decreasing, tol) if stepper is None else stepper
    losses = []
    while st.continual:
        P = S @ A[:, :, :3].transpose(0, 2, 1) + A[:, None, :, 3]
        err = np.empty(B)
        M = np.empty_like(P)
        for b in range(B):
            d, j = nearest(P[b], Tg[b], ord, matcher)
            err[b] = d.mean()
            M[b] = Tg[b][j]
        for b in range(B):
            ms, mt = P[b].mean(0), M[b].mean(0)
            R = kabsch((M[b] - mt).T @ (P[b] - ms), eps)
            t = mt - R @ ms
            A[b] = np.concatenate([R @ A[b, :, :3], (R @ A[b, :, 3] + t)[:, None]], 1)
        losses.append(err)
        st.step(err)
    return A, np.array(losses), batch
