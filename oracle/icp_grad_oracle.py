"""fp64 torch-autograd model of the reference's ICP graph (pypose/module/icp.py:73-110), for the ICP gradient tests.

Test infrastructure only: the package never imports it.  It rebuilds the graph from its definition, on any device:
* per iteration: k = 1 matching (no gradient; or the matches the caller gives), gather, svdtf (centroids, H,
  torch.linalg.svd, U @ Vh negated as a whole when det = -1, t = mt - R ms), the quaternion of mat2SE3, and SE3 Act;
* SE3 Act backward gives the 7-vector of T the gradient [sum g, sum out x g, 0] and the points R^T g;
* the closing svdtf(source, p_K), whose quaternion takes the sign rule `final`: "reference" (mat2SE3's) or "project"
  (w >= 0, what pp.module.ICP returns);
* the iteration count is given (K), so the graph is that of a run with K iterations.
"""
import torch


def quat2mat(q):
    x, y, z, w = q.unbind(-1)
    return torch.stack([
        torch.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z], -1)], -2)


def mat2quat_ref(R):
    """mat2SE3's quaternion [x y z w]: branch on R22 < 1e-5, then R00 > R11 (or R00 < -R11); w keeps its branch's sign.
    Only the chosen branch is differentiated (the others are multiplied by 0, with finite square roots)."""
    r = lambda i, j: R[..., i, j]   # noqa: E731
    d2 = r(2, 2) < 1e-5
    c0 = d2 & (r(0, 0) > r(1, 1))
    c1 = d2 & ~(r(0, 0) > r(1, 1))
    c2 = ~d2 & (r(0, 0) < -r(1, 1))
    c3 = ~d2 & ~(r(0, 0) < -r(1, 1))
    t0 = 1 + r(0, 0) - r(1, 1) - r(2, 2)
    t1 = 1 - r(0, 0) + r(1, 1) - r(2, 2)
    t2 = 1 - r(0, 0) - r(1, 1) + r(2, 2)
    t3 = 1 + r(0, 0) + r(1, 1) + r(2, 2)
    q0 = torch.stack([t0, r(1, 0) + r(0, 1), r(0, 2) + r(2, 0), r(2, 1) - r(1, 2)], -1)
    q1 = torch.stack([r(1, 0) + r(0, 1), t1, r(2, 1) + r(1, 2), r(0, 2) - r(2, 0)], -1)
    q2 = torch.stack([r(0, 2) + r(2, 0), r(2, 1) + r(1, 2), t2, r(1, 0) - r(0, 1)], -1)
    q3 = torch.stack([r(2, 1) - r(1, 2), r(0, 2) - r(2, 0), r(1, 0) - r(0, 1), t3], -1)
    m = [c.to(R.dtype) for c in (c0, c1, c2, c3)]
    q = sum(qi * mi.unsqueeze(-1) for qi, mi in zip((q0, q1, q2, q3), m))
    t = sum(ti * mi for ti, mi in zip((t0, t1, t2, t3), m))
    return q / (2 * torch.sqrt(t)).unsqueeze(-1)


class Act(torch.autograd.Function):
    """SE3 Act of X (..., 7) on points p (..., 3) with the reference's backward convention."""

    @staticmethod
    def forward(ctx, X, p):
        R = quat2mat(X[..., 3:])
        out = (R @ p.unsqueeze(-1)).squeeze(-1) + X[..., :3]
        ctx.save_for_backward(R, out)
        return out

    @staticmethod
    def backward(ctx, g):
        R, out = ctx.saved_tensors
        gX = torch.cat([g, torch.linalg.cross(out, g), torch.zeros_like(g[..., :1])], -1)
        return gX, (R.mT @ g.unsqueeze(-1)).squeeze(-1)


class Matrix(torch.autograd.Function):
    """The 4x4 matrix of X (..., 7) with the reference's convention (Act on the rows of I4, transposed): the 7-vector
    gets [W_t, sum_j col_j x W_j, 0] for the cotangent W of the matrix."""

    @staticmethod
    def forward(ctx, X):
        M = torch.zeros(X.shape[:-1] + (4, 4), dtype=X.dtype, device=X.device)
        M[..., :3, :3] = quat2mat(X[..., 3:])
        M[..., :3, 3] = X[..., :3]
        M[..., 3, 3] = 1
        ctx.save_for_backward(M)
        return M

    @staticmethod
    def backward(ctx, W):
        M, = ctx.saved_tensors
        cols, g = M[..., :3, :].mT, W[..., :3, :].mT          # (..., 4, 3): out_j and its cotangent
        om = torch.linalg.cross(cols, g).sum(-2)
        return torch.cat([W[..., :3, 3], om, torch.zeros_like(om[..., :1])], -1)


def svdtf(source, target, final=None):
    """The reference's svdtf as a 7-vector; final="project" flips q to w >= 0."""
    cs, ct = source.mean(-2, keepdim=True), target.mean(-2, keepdim=True)
    H = torch.einsum("...na,...nb->...ab", target - ct, source - cs)
    U, S, Vh = torch.linalg.svd(H)
    R = U @ Vh
    neg = ((torch.linalg.det(R) + 1).abs() < 1e-6).to(R.dtype)[..., None, None]
    R = R * (1 - 2 * neg)
    t = ct.mT - R @ cs.mT
    q = mat2quat_ref(R)
    if final == "project":
        q = q * torch.where(q[..., 3:] < 0, -1.0, 1.0).to(q.dtype)
    return torch.cat([t.squeeze(-1), q], -1)


def _dist(a, b, ord):
    d = a[..., :, None, :] - b[..., None, :, :]
    if ord == 2:
        return d.square().sum(-1)
    if ord == 1:
        return d.abs().sum(-1)
    return d.abs().amax(-1)


def icp(source, target, K, init=None, ord=2, final="project", matches=None):
    """The reference's ICP graph with K iterations: returns the 7-vector (batch, 7) and the per-iteration matches.
    matches: K index tensors (batch, Ns) that iteration k gathers instead of matching (the graph is otherwise the same),
    so that a run whose nearest neighbours were decided elsewhere (in fp32, say) can be replayed exactly."""
    batch = torch.broadcast_shapes(source.shape[:-2], target.shape[:-2], *([init.shape[:-1]] if init is not None else []))
    temporal = source if init is None else Act.apply(init.unsqueeze(-2), source)
    temporal = temporal.expand(batch + source.shape[-2:])
    tgt = target.expand(batch + target.shape[-2:])
    if matches is not None and len(matches) != K:
        raise ValueError(f"icp: {len(matches)} match tensors for K = {K}")
    used = []
    for k in range(K):
        if matches is not None:
            idx = matches[k].to(device=tgt.device, dtype=torch.long).reshape(batch + source.shape[-2:-1])
        else:
            with torch.no_grad():
                idx = _dist(temporal, tgt, ord).argmin(-1)   # ties: the first (lowest) index
        used.append(idx)
        knn = torch.gather(tgt, -2, idx.unsqueeze(-1).expand(idx.shape + (3,)))
        T = svdtf(temporal, knn)
        temporal = Act.apply(T.unsqueeze(-2), temporal)
    return svdtf(source.expand(batch + source.shape[-2:]), temporal, final), used


def losses(T, W, probe, w):
    """The two test losses on a 7-vector T (batch, 7): sum W * matrix(T), sum w . T Act probe."""
    return (Matrix.apply(T) * W).sum(), (Act.apply(T.unsqueeze(-2), probe) * w).sum()


def grads(source, target, K, init=None, ord=2, final="project", W=None, probe=None, w=None, which=0, matches=None):
    """Gradients of loss `which` (0: matrix, 1: Act) w.r.t. source, target and init (None where not given); matches as
    in icp()."""
    leaves = [x.detach().clone().requires_grad_() if x is not None else None for x in (source, target, init)]
    T, _ = icp(leaves[0], leaves[1], K, leaves[2], ord, final, matches)
    L = losses(T, W, probe, w)[which]
    gs = torch.autograd.grad(L, [x for x in leaves if x is not None])
    it = iter(gs)
    return T.detach(), [next(it) if x is not None else None for x in leaves]


def sign_agrees(R):
    """True where mat2SE3's quaternion of R already has w >= 0 (the two sign rules agree)."""
    return mat2quat_ref(R)[..., 3] >= 0

