"""Linear quadratic regulator (reference: pypose/module/lqr.py).  DESIGN.md §3.7.

Two routes, chosen per call from the system:

* affine route (csrc/lqr.cu): the system is an `LTI` or `LTV` whose class keeps the base `forward`,
  `state_transition` and `set_refpoint`, n = ns + nc <= 32, and the tensors are on CUDA.  One launch per call solves every problem of the batch
  (one warp per problem), and one more solves the KKT adjoint in the backward pass.  A time-invariant operand is read
  from one copy through a zero stride.  An `LTV` subclass that overrides `A`, `B` or `c1` has them gathered per step, if
  the reference's three system-time sequences coincide (system time 0 on entry and int(t * dt) == t);
* generic route: every other system, CPU tensors and inputs the reference rejects, with the reference's algorithm in
  torch ops.
"""
from typing import Optional

import torch
from torch import Tensor, nn

from .. import _C
from ..function.linalg import bmv, bvmv
from .dynamics import LTI, LTV, runsys

_BASE_METHODS = ('forward', 'state_transition', 'set_refpoint')


def _strides(t, inner):
    """element strides of the (batch, step) axes of a compact (nb|1, T|1, ...) operand; 0 where the axis has size 1"""
    return (0 if t.shape[0] == 1 else t[0].numel()), (0 if t.shape[1] == 1 else inner)


def _launch_args(Q, p, A, B, c1, x_init, u_traj):
    n, ns = p.shape[-1], x_init.shape[-1]
    nc = n - ns
    args = []
    for t, inner in ((Q, n * n), (p, n), (A, ns * ns), (B, ns * nc), (c1, ns)):
        args += [0, 0, 0] if t is None else [t.data_ptr(), *_strides(t, inner)]
    args.append(x_init.data_ptr())
    args += [0, 0, 0] if u_traj is None else [u_traj.data_ptr(), *_strides(u_traj, nc)]
    return args


def _check(Q, p, A, B, c1, x_init, u_traj, T):
    """every operand reaches the kernel as a raw pointer read through strides: shapes, device and dtype are checked
    here, so that no step or problem is read past the end of its buffer"""
    if x_init.ndim != 2 or p.ndim != 3 or T < 1:
        raise ValueError(f"lqr_affine: expected x_init (nb, ns), p (nb|1, T|1, n) and T >= 1, got {tuple(x_init.shape)}, "
                         f"{tuple(p.shape)}, T = {T}")
    nb, ns = x_init.shape
    n = p.shape[-1]
    nc = n - ns
    if not (1 <= ns < n <= 32):
        raise ValueError(f"lqr_affine: needs 1 <= ns < n = ns + nc <= 32, got ns = {ns}, n = {n}")
    for name, t, tail in (("Q", Q, (n, n)), ("p", p, (n,)), ("A", A, (ns, ns)), ("B", B, (ns, nc)), ("c1", c1, (ns,)),
                          ("u_traj", u_traj, (nc,))):
        if t is None:
            continue
        if (t.ndim != 2 + len(tail) or t.shape[0] not in (1, nb) or t.shape[1] not in (1, T)
                or tuple(t.shape[2:]) != tail):
            raise ValueError(f"lqr_affine: {name} must be (nb|1, T|1, {', '.join(map(str, tail))}) with nb = {nb}, "
                             f"T = {T}, got {tuple(t.shape)}")
        if t.device != x_init.device or t.dtype != x_init.dtype:
            raise ValueError(f"lqr_affine: {name} is on {t.device} / {t.dtype}, x_init on {x_init.device} / "
                             f"{x_init.dtype}")


@torch.library.custom_op("b200pose::lqr_affine", mutates_args=(), device_types="cuda")
def lqr_affine(Q: Tensor, p: Tensor, A: Tensor, B: Tensor, c1: Optional[Tensor], x_init: Tensor,
               u_traj: Optional[Tensor], T: int) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Batched LQR for x' = A_t x + B_t u + c1_t.  Operands are contiguous and compact: Q (nb|1, T|1, n, n),
    p (nb|1, T|1, n), A (nb|1, T|1, ns, ns), B (nb|1, T|1, ns, nc), c1 (nb|1, T|1, ns) or None, x_init (nb, ns),
    u_traj (nb|1, T|1, nc) or None; an axis of size 1 is broadcast.  Returns x (nb, T+1, ns), u (nb, T, nc), cost (nb),
    x_traj (nb, T, ns) and an int32 status (nb), 1 where a Quu is not positive definite."""
    _check(Q, p, A, B, c1, x_init, u_traj, T)
    Q, p, A, B, x_init = (t.contiguous() for t in (Q, p, A, B, x_init))
    c1 = None if c1 is None else c1.contiguous()
    u_traj = None if u_traj is None else u_traj.contiguous()
    nb, ns = x_init.shape
    n = p.shape[-1]
    nc = n - ns
    x, u = x_init.new_empty(nb, T + 1, ns), x_init.new_empty(nb, T, nc)
    cost, xtr = x_init.new_empty(nb), x_init.new_empty(nb, T, ns)
    status = torch.zeros(nb, dtype=torch.int32, device=x_init.device)
    ws = x_init.new_empty(nb * T * nc * (ns + 1))
    _C.enqueue(f"b200_lqr_affine_{_C.suffix(x_init.dtype)}", x_init, *_launch_args(Q, p, A, B, c1, x_init, u_traj),
               x.data_ptr(), u.data_ptr(), cost.data_ptr(), xtr.data_ptr(), status.data_ptr(), ws.data_ptr(), nb, T, ns,
               nc)
    return x, u, cost, xtr, status


@lqr_affine.register_fake
def _(Q, p, A, B, c1, x_init, u_traj, T):
    nb, ns = x_init.shape
    nc = p.shape[-1] - ns
    return (x_init.new_empty(nb, T + 1, ns), x_init.new_empty(nb, T, nc), x_init.new_empty(nb),
            x_init.new_empty(nb, T, ns), x_init.new_empty(nb, dtype=torch.int32))


@torch.library.custom_op("b200pose::lqr_affine_bwd", mutates_args=(), device_types="cuda")
def lqr_affine_bwd(Q: Tensor, p: Tensor, A: Tensor, B: Tensor, c1: Optional[Tensor], x_init: Tensor, T: int, x: Tensor,
                   u: Tensor, gx: Tensor, gu: Tensor, gcost: Tensor) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """KKT adjoint of `lqr_affine` at its solution (x, u): gradients with respect to Q (symmetric), p, A, B, c1 (empty
    when c1 is None) and x_init, per problem (nb, T|1, ...) with the step axis of the operand (summed when it is 1)."""
    _check(Q, p, A, B, c1, x_init, None, T)
    nb, ns = x_init.shape
    nc = p.shape[-1] - ns
    for t, shape in ((x, (nb, T + 1, ns)), (u, (nb, T, nc)), (gx, (nb, T + 1, ns)), (gu, (nb, T, nc)), (gcost, (nb,))):
        if tuple(t.shape) != shape or t.device != x_init.device or t.dtype != x_init.dtype:
            raise ValueError(f"lqr_affine_bwd: expected {shape} on {x_init.device} / {x_init.dtype}, got "
                             f"{tuple(t.shape)} on {t.device} / {t.dtype}")
    Q, p, A, B, x_init, x, u, gx, gu, gcost = (t.contiguous() for t in (Q, p, A, B, x_init, x, u, gx, gu, gcost))
    c1 = None if c1 is None else c1.contiguous()
    nb, ns = x_init.shape
    n = p.shape[-1]
    nc = n - ns
    grads, flags = [], []
    for t in (Q, p, A, B, c1):
        if t is None:
            grads.append(x_init.new_empty(0))
            flags.append(0)
            continue
        grads.append(x_init.new_empty(nb, t.shape[1], *t.shape[2:]))
        flags.append(int(t.shape[1] != 1 or T == 1))
    gx0 = x_init.new_empty(nb, ns)
    ws = x_init.new_empty(nb * T * (nc * (ns + 1) + n))
    out = []
    for g, f, t in zip(grads, flags, (Q, p, A, B, c1)):
        out += [g.data_ptr() if t is not None else 0, f]
    _C.enqueue(f"b200_lqr_affine_bwd_{_C.suffix(x_init.dtype)}", x_init,
               *_launch_args(Q, p, A, B, c1, x_init, None), x.data_ptr(), u.data_ptr(), gx.data_ptr(), gu.data_ptr(),
               gcost.data_ptr(), *out, gx0.data_ptr(), ws.data_ptr(), nb, T, ns, nc)
    return (*grads, gx0)


@lqr_affine_bwd.register_fake
def _(Q, p, A, B, c1, x_init, T, x, u, gx, gu, gcost):
    nb = x_init.shape[0]
    g = [x_init.new_empty(0) if t is None else x_init.new_empty(nb, *t.shape[1:]) for t in (Q, p, A, B, c1)]
    return (*g, x_init.new_empty(x_init.shape))


def _setup(ctx, inputs, output):
    Q, p, A, B, c1, x_init, u_traj, T = inputs
    ctx.save_for_backward(Q, p, A, B, c1, x_init, output[0], output[1])
    ctx.T = T
    ctx.mark_non_differentiable(output[3], output[4])


def _backward(ctx, gx, gu, gcost, _gxtr, _gst):
    Q, p, A, B, c1, x_init, x, u = ctx.saved_tensors
    z = lambda g, ref: torch.zeros_like(ref) if g is None else g.contiguous()   # noqa: E731
    grads = torch.ops.b200pose.lqr_affine_bwd(Q, p, A, B, c1, x_init, ctx.T, x, u, z(gx, x), z(gu, u),
                                              z(gcost, x[:, 0, 0]))
    out = []
    for g, t in zip(grads[:5], (Q, p, A, B, c1)):
        if t is None:
            out.append(None)
            continue
        out.append(g.sum(0, keepdim=True) if t.shape[0] == 1 and g.shape[0] != 1 else g)
    return (*out, grads[5], None, None)


lqr_affine.register_autograd(_backward, setup_context=_setup)


def _compact(t, lead):
    """(nb, T, ...) with zero-stride (expanded) leading axes -> a contiguous operand whose broadcast axes have size 1"""
    for d in range(lead):
        if t.shape[d] > 1 and t.stride(d) == 0:
            t = t.narrow(d, 0, 1)
    return t.contiguous()


class LQR(nn.Module):
    r"""Linear quadratic regulator by dynamic programming.

    Args:
        system: the dynamics (`LTI`, `LTV`, `NLS` or any `System`).
        Q (Tensor): quadratic weights, (nb, T, n, n) or (nb, n, n) shared over the steps; n = ns + nc.
        p (Tensor): linear weights, (nb, T, n) or (nb, n).
        T (int): the horizon.

    `forward(x_init, dt=1, u_traj=None, u_lower=None, u_upper=None, du=None)` returns the states x (nb, T+1, ns), the
    inputs u (nb, T, nc) and the costs (nb) of the minimiser of sum_t tau_t^T Q_t tau_t / 2 + p_t^T tau_t, tau_t =
    [x_t; u_t], subject to the dynamics, linearised around the rollout of `u_traj` (zeros when None).  `u_lower`,
    `u_upper` and `du` are accepted and ignored, as in the reference.  The rollout is left on `x_traj`, the inputs it
    used on `u_traj`.

    For an `LTI` or `LTV` on CUDA tensors with n <= 32 the solve and its backward pass are CUDA kernels (module
    docstring); there a
    `Quu` that is not positive definite raises `torch.linalg.LinAlgError` after one read of the per-problem status, the
    gradient with respect to Q is its symmetric part, `x_traj` carries no gradient and the gradient with respect to
    `u_traj` is zero (the minimiser does not depend on it).  The generic route applies the reference's `squeeze(-2)`
    to linearised matrices only when they carry the Jacobian's extra batch axis, so a 1x1 state matrix is kept.
    """

    def __init__(self, system, Q, p, T):
        super().__init__()
        self.system = system
        self.Q, self.p, self.T = Q, p, T
        self.x_traj = None
        self.u_traj = None
        if self.Q.ndim == 3:
            self.Q = self.Q.clone().unsqueeze(-3).expand(-1, self.T, -1, -1)
        if self.p.ndim == 2:
            self.p = self.p.clone().unsqueeze(-2).expand(-1, self.T, -1)
        self.n_batch = self.p.shape[:-2]
        assert self.Q.shape[:-1] == self.p.shape, "Shape not compatible."
        assert self.Q.size(-1) == self.Q.size(-2), "Shape not compatible."
        assert self.Q.ndim == 4 or self.p.ndim == 3, "Shape not compatible."
        assert self.Q.device == self.p.device, "Device not compatible."
        assert self.Q.dtype == self.p.dtype, "Tensor data type not compatible."
        self.dargs = {'dtype': self.p.dtype, 'device': self.p.device}

    def forward(self, x_init, dt=1, u_traj=None, u_lower=None, u_upper=None, du=None):
        route = self._route(x_init, dt, u_traj)
        if route is not None:
            return self._affine(x_init, dt, u_traj, route)
        K, k = self.lqr_backward(x_init, dt, u_traj, u_lower, u_upper, du)
        return self.lqr_forward(x_init, K, k, u_lower, u_upper, du)

    # ------------------------------------------------------------------------------------------------ affine route
    def _route(self, x_init, dt, u_traj):
        """'lti', 'ltv' (matrices independent of the system time), 'gather' (per-step properties of an LTV) or None for
        the generic route.  Inputs the reference rejects (Q / p with a step axis other than T, mismatched devices or
        dtypes) take the generic route, which raises as the reference does; so do tensors off CUDA, where the generic
        route is plain torch."""
        sys, cls = self.system, type(self.system)
        if not isinstance(sys, LTI):
            return None
        base = LTV if isinstance(sys, LTV) else LTI
        if any(getattr(cls, m) is not getattr(base, m) for m in _BASE_METHODS):
            return None
        n, ns = self.p.size(-1), x_init.size(-1)
        if not (1 <= ns < n <= 32) or x_init.ndim != 2 or len(self.n_batch) != 1 or x_init.shape[0] != self.n_batch[0]:
            return None
        if self.Q.ndim != 4 or self.Q.shape[-3] != self.T or self.p.shape[-2] != self.T:
            return None
        if not x_init.is_cuda or x_init.device != self.p.device:
            return None
        if x_init.dtype not in (torch.float32, torch.float64) or x_init.dtype != self.p.dtype:
            return None
        if u_traj is not None and (u_traj.shape != self.n_batch + (self.T, n - ns) or u_traj.device != x_init.device
                                   or u_traj.dtype != x_init.dtype):
            return None
        if any(getattr(cls, a) is not getattr(LTI, a) for a in ('A', 'B', 'c1')):
            # an LTV's properties are read at the system time its set_refpoint sets; for other LTI subclasses the
            # reference reads them at times that differ between its three passes
            if base is not LTV or int(sys.systime) != 0 or any(int(t * dt) != t for t in range(self.T)):
                return None
            return 'gather'
        return 'ltv' if base is LTV else 'lti'

    def _operand(self, m, shape):
        """a system matrix (..., *shape) with no or one batch axis -> (nb|1, 1, *shape), or None when it does not fit"""
        if m is None:
            return None
        if m.ndim == len(shape):
            m = m.unsqueeze(0)
        if m.ndim != len(shape) + 1 or tuple(m.shape[1:]) != shape or m.shape[0] not in (1, self.n_batch[0]):
            raise ValueError
        return m.unsqueeze(1)

    def _affine(self, x_init, dt, u_traj, route):
        sys, T = self.system, self.T
        nb, ns = x_init.shape
        nc = self.p.size(-1) - ns
        s0 = int(sys.systime)
        try:
            if route == 'gather':
                mats = []
                for t in range(T):
                    sys.systime = t
                    mats.append((self._operand(sys.A, (ns, ns)), self._operand(sys.B, (ns, nc)),
                                 self._operand(sys.c1, (ns,))))
                A, B, c1 = (None if mats[0][i] is None else
                            torch.cat(torch.broadcast_tensors(*[m[i] for m in mats]), 1) for i in range(3))
            else:
                A, B, c1 = (self._operand(sys.A, (ns, ns)), self._operand(sys.B, (ns, nc)),
                            self._operand(sys.c1, (ns,)))
            dev, dt_ = x_init.device, x_init.dtype
            if any(m is not None and (m.device != dev or m.dtype != dt_) for m in (A, B, c1)):
                raise ValueError
        except ValueError:
            sys.systime = s0
            K, k = self.lqr_backward(x_init, dt, u_traj)
            return self.lqr_forward(x_init, K, k)
        self.u_traj = torch.zeros(self.n_batch + (T, nc), **self.dargs) if u_traj is None else u_traj
        x, u, cost, xtr, status = torch.ops.b200pose.lqr_affine(
            _compact(self.Q, 2), _compact(self.p, 2), A.contiguous(), B.contiguous(),
            None if c1 is None else c1.contiguous(), x_init.contiguous(),
            None if u_traj is None else _compact(u_traj, 2), T)
        if bool(status.any()):
            raise torch.linalg.LinAlgError("LQR: Quu is not positive definite (cholesky failed)")
        self.x_traj = xtr
        sys.systime = s0 + 2 * T - 1 if route == 'lti' else (T if T >= 2 or route == 'gather' else s0 + 1)
        sys.state, sys.input = x[..., T - 1, :], u[..., T - 1, :]
        return x, u, cost

    # ----------------------------------------------------------------------------------------------- generic route
    def lqr_backward(self, x_init, dt, u_traj=None, u_lower=None, u_upper=None, du=None):
        ns, nsc = x_init.size(-1), self.p.size(-1)
        nc = nsc - ns
        self.u_traj = torch.zeros(self.n_batch + (self.T, nc), **self.dargs) if u_traj is None else u_traj
        self.x_traj = runsys(self.system, self.T, x_init.unsqueeze(-2).repeat((1, self.T, 1)), self.u_traj)
        K = torch.zeros(self.n_batch + (self.T, nc, ns), **self.dargs)
        k = torch.zeros(self.n_batch + (self.T, nc), **self.dargs)
        p = bmv(self.Q, torch.cat((self.x_traj[..., :self.T, :], self.u_traj), dim=-1)) + self.p
        V = v = None
        for t in range(self.T - 1, -1, -1):
            Qt, qt = self.Q[..., t, :, :], p[..., t, :]
            if t < self.T - 1:
                self.system.set_refpoint(state=self.x_traj[..., t, :], input=self.u_traj[..., t, :],
                                         t=torch.tensor(t * dt))
                A, B = self.system.A, self.system.B
                if A.ndim > 3:               # the Jacobian's extra batch axis of a linearised system
                    A, B = A.squeeze(-2), B.squeeze(-2)
                F = torch.cat((A, B), dim=-1)
                Qt = Qt + F.mT @ V @ F
                qt = qt + bmv(F.mT, v)
            Qxx, Qxu, Qux, Quu = Qt[..., :ns, :ns], Qt[..., :ns, ns:], Qt[..., ns:, :ns], Qt[..., ns:, ns:]
            qx, qu = qt[..., :ns], qt[..., ns:]
            L = torch.linalg.cholesky(Quu)
            K[..., t, :, :] = Kt = -torch.cholesky_solve(Qux, L)
            k[..., t, :] = kt = -torch.cholesky_solve(qu.unsqueeze(-1), L).squeeze(-1)
            V = Qxx + Qxu @ Kt + Kt.mT @ Qux + Kt.mT @ Quu @ Kt
            v = qx + bmv(Qxu, kt) + bmv(Kt.mT, qu) + bmv(Kt.mT @ Quu, kt)
        return K, k

    def lqr_forward(self, x_init, K, k, u_lower=None, u_upper=None, du=None):
        assert x_init.device == K.device == k.device
        assert x_init.dtype == K.dtype == k.dtype
        assert x_init.ndim == 2, "Shape not compatible."
        ns, nc = self.x_traj.size(-1), self.u_traj.size(-1)
        u = torch.zeros(self.n_batch + (self.T, nc), **self.dargs)
        cost = torch.zeros(self.n_batch, **self.dargs)
        x = torch.zeros(self.n_batch + (self.T + 1, ns), **self.dargs)
        xt = x[..., 0, :] = x_init
        for t in range(self.T):
            u[..., t, :] = ut = bmv(K[..., t, :, :], xt - self.x_traj[..., t, :]) + k[..., t, :] + self.u_traj[..., t, :]
            xut = torch.cat((xt, ut), dim=-1)
            x[..., t + 1, :] = xt = self.system(xt, ut)[0]
            cost = cost + 0.5 * bvmv(xut, self.Q[..., t, :, :], xut) + torch.linalg.vecdot(xut, self.p[..., t, :])
        return x, u, cost
