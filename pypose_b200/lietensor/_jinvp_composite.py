"""Gradient of Jinvp with respect to the group element (rare path).

The reference has no custom backward for Jinvp: autograd differentiates through Log and the
explicit Jl^-1 matrix build (lietensor.py:261, 426, 560, 704).  The hot path never needs this
gradient, so instead of a kernel we differentiate a composite built from torch matrix ops and our
own differentiable Log op.  so3/se3/rxso3 use the closed-form Jl^-1 (operation.py:23-32, 68-75,
137-140) with series coefficients near theta = 0; sim3 uses the truncated series (operation.py:167-172).
"""
import torch

from .basics import vec2skew


def _coef(theta2, closed, series):
    small = theta2 < 1e-4
    safe = torch.where(small, torch.ones_like(theta2), theta2)
    return torch.where(small, series(theta2), closed(safe))


def _so3_jlinv(phi):
    K = vec2skew(phi)
    t2 = (phi * phi).sum(-1)[..., None, None]

    def closed(x):
        th = x.sqrt()
        return (1 - 0.5 * th * torch.cos(0.5 * th) / torch.sin(0.5 * th)) / x
    c = _coef(t2, closed, lambda x: 1 / 12 + x / 720 + x * x / 30240)
    I = torch.eye(3, dtype=phi.dtype, device=phi.device).expand(phi.shape[:-1] + (3, 3))
    return I - 0.5 * K + c * (K @ K)


def _calcQ(tau, phi):
    T, P = vec2skew(tau), vec2skew(phi)
    t2 = (phi * phi).sum(-1)[..., None, None]

    def c1(x):
        th = x.sqrt()
        return (th - th.sin()) / (x * th)

    def c2(x):
        th = x.sqrt()
        return (x + 2 * th.cos() - 2) / (2 * x * x)

    def c3(x):
        th = x.sqrt()
        return (2 * th - 3 * th.sin() + th * th.cos()) / (2 * x * x * th)
    a1 = _coef(t2, c1, lambda x: 1 / 6 - x / 120 + x * x / 5040)
    a2 = _coef(t2, c2, lambda x: 1 / 24 - x / 720 + x * x / 40320)
    a3 = _coef(t2, c3, lambda x: 1 / 120 - x / 2520 + x * x / 120960)
    return (0.5 * T + a1 * (P @ T + T @ P + P @ T @ P) + a2 * (P @ P @ T + T @ P @ P - 3 * P @ T @ P)
            + a3 * (P @ T @ P @ P + P @ P @ T @ P))


def _sim3_ad(x):
    tau, phi, sigma = x[..., :3], x[..., 3:6], x[..., 6:]
    I = torch.eye(3, dtype=x.dtype, device=x.device)
    top = torch.cat([vec2skew(phi) + sigma[..., None] * I, vec2skew(tau), -tau[..., None]], -1)
    mid = torch.cat([torch.zeros_like(top[..., :3]), vec2skew(phi), torch.zeros_like(tau[..., None])], -1)
    return torch.cat([top, mid, torch.zeros_like(top[..., :1, :])], -2)


def jlinv_times(grp, x, p):
    if grp == "SO3":
        return (_so3_jlinv(x) @ p[..., None])[..., 0]
    if grp == "RxSO3":
        return torch.cat([(_so3_jlinv(x[..., :3]) @ p[..., :3, None])[..., 0], p[..., 3:]], -1)
    if grp == "SE3":
        Ji, Q = _so3_jlinv(x[..., 3:]), _calcQ(x[..., :3], x[..., 3:])
        hr = (Ji @ p[..., 3:, None])
        ht = Ji @ (p[..., :3, None] - Q @ hr)
        return torch.cat([ht[..., 0], hr[..., 0]], -1)
    Xi = _sim3_ad(x)
    Xi2 = Xi @ Xi
    M = torch.eye(7, dtype=x.dtype, device=x.device) - Xi / 2 + Xi2 / 12 - (Xi2 @ Xi2) / 720
    return (M @ p[..., None])[..., 0]


def grad_X(grp, X, p, g):
    """Left-tangent gradient of g . Jinvp(X, p) with respect to X, evaluated in fp64 for every input dtype: in fp32 the
    closed-form coefficients lose their digits just above the series switch (c2's numerator theta^2 + 2 cos(theta) - 2
    is theta^4 / 12, below fp32's rounding of cos(theta) for theta < 0.03), and their autograd derivative, divided by
    theta^2, turns that into gradient errors of 1e-2 at theta = 0.01."""
    from .ops import _apply
    with torch.enable_grad():
        Xd = X.detach().double().requires_grad_(True)
        x = _apply(f"{grp}_log_fwd", Xd)
        out = jlinv_times(grp, x, p.detach().double())
        (gX,) = torch.autograd.grad(out, Xd, g.double())
    return gX.to(X.dtype)
