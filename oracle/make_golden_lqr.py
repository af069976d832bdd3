"""Write tests/golden/lqr.npz from the reference pp.module.LQR / MPC on the CPU (PYPOSE_REFERENCE names a pypose v0.9.5
checkout).  Each case stores its seeded inputs, the reference's fp64 x / u / cost, and the relative error of the same
reference run in fp32 against them (`err32`, max |a - b| / max |b| per output).  For `grad` cases it also stores the
reference's fp64 autograd gradients of <gx, x> + <gu, u> + <gc, cost> under a seeded cotangent.  `indefinite` is a case
where the reference's cholesky raises.

The reference cannot solve a system with ns = 1: its `A.squeeze(-2)` collapses the 1x1 state matrix.  The ns = nc = 1
case (`from: oracle`) therefore stores the fp64 oracle's solution (oracle/lqr_oracle.py) and, as its fp32 yardstick,
the error of the reference's algorithm in torch ops run in fp32 (pypose_b200's generic LQR route, which differs from the
reference only in keeping that matrix).

`cartpole_lqr` / `cartpole_mpc` solve the standard cart-pole (an NLS, written below) with LQR and with MPC under
ReduceToBason(10); they take the generic route.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
import pypose as pp  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "lqr.npz")
D = torch.float64


def spd(g, *shape, n):
    M = torch.randn(*shape, n, n, generator=g, dtype=D)
    return M.mT @ M + 0.5 * torch.eye(n, dtype=D)


class StepLTV(pp.module.LTV):
    """per-step A_t, B_t read at the system time"""
    @property
    def A(self):
        return self._A[:, int(self._t)]

    @property
    def B(self):
        return self._B[:, int(self._t)]


def case(seed, nb, T, ns, nc, q_step=True, p3=True, c1=True, u=False, ltv=False, dt=1, grad=False, indefinite=False):
    g = torch.Generator().manual_seed(seed)
    n = ns + nc
    Q = spd(g, nb, *((T,) if q_step else ()), n=n)
    if indefinite:
        Q[0, ..., ns:, ns:] -= 100 * torch.eye(nc, dtype=D)
    p = torch.randn(nb, *((T,) if p3 else ()), n, generator=g, dtype=D)
    At = 0.8 * torch.eye(ns, dtype=D) + 0.2 / ns ** 0.5 * torch.randn(nb, *((T,) if ltv else ()), ns, ns, generator=g, dtype=D)
    Bt = torch.randn(nb, *((T,) if ltv else ()), ns, nc, generator=g, dtype=D)
    c1t = torch.randn(nb, ns, generator=g, dtype=D) if c1 else None
    x0 = torch.randn(nb, ns, generator=g, dtype=D)
    ut = torch.randn(nb, T, nc, generator=g, dtype=D) if u else None
    ins = dict(Q=Q, p=p, A=At, B=Bt, c1=c1t, x0=x0, u_traj=ut)
    leaves = {k: v.clone().requires_grad_(grad) for k, v in ins.items() if v is not None}
    C, Dm = torch.eye(ns, dtype=D).expand(nb, ns, ns), torch.zeros(nb, ns, nc, dtype=D)
    cls = StepLTV if ltv else pp.module.LTI
    sys_ = cls(leaves["A"], leaves["B"], C, Dm, leaves.get("c1"), None)
    out = {k: v.numpy() for k, v in ins.items() if v is not None}
    meta = dict(kind="ltv" if ltv else "lti", nb=nb, T=T, ns=ns, nc=nc, ltv=ltv, dt=dt, c1=c1, u=u, grad=grad,
                raises=False, **{"from": "reference"})
    if ns == 1:
        return oracle_case(meta, ins, out)
    try:
        x, uu, cost = pp.module.LQR(sys_, leaves["Q"], leaves["p"], T)(leaves["x0"], dt, leaves.get("u_traj"))
    except torch.linalg.LinAlgError:
        meta["raises"] = True
        return meta, out
    meta["systime"] = int(sys_.systime)
    out.update(x=x.detach().numpy(), u=uu.detach().numpy(), cost=cost.detach().numpy())
    f = {k: None if v is None else v.float() for k, v in ins.items()}
    C32, D32 = C.float(), Dm.float()
    x32, u32, c32 = pp.module.LQR(cls(f["A"], f["B"], C32, D32, f["c1"], None), f["Q"], f["p"], T)(f["x0"], dt, f["u_traj"])
    meta["err32"] = err32((x32, u32, c32), out)
    if grad:
        gx, gu, gc = (torch.randn(t.shape, generator=g, dtype=D) for t in (x, uu, cost))
        names = [k for k in ("Q", "p", "A", "B", "c1", "x0") if k in leaves]
        gr = torch.autograd.grad((x * gx).sum() + (uu * gu).sum() + (cost * gc).sum(), [leaves[k] for k in names])
        out.update(gx=gx.numpy(), gu=gu.numpy(), gc=gc.numpy())
        out.update({f"g{k}": v.numpy() for k, v in zip(names, gr)})
    return meta, out


def err32(outs32, out):
    return {k: float(np.abs(o.detach().double().numpy() - out[k]).max() / np.abs(out[k]).max())
            for k, o in zip(("x", "u", "cost"), outs32)}


def oracle_case(meta, ins, out):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import lqr_oracle as O
    import pypose_b200 as pb
    meta["from"] = "oracle"
    n = lambda k: None if ins[k] is None else ins[k].numpy()   # noqa: E731
    nb, T = meta["nb"], meta["T"]
    Q, p = n("Q"), n("p")
    Q, p = (Q if Q.ndim == 4 else Q[:, None]), (p if p.ndim == 3 else p[:, None])
    F = O.full(Q, p, n("A")[:, None], n("B")[:, None], None if ins["c1"] is None else n("c1")[:, None], n("x0"), n("u_traj"))
    F = [np.broadcast_to(a, (nb, T) + a.shape[2:]) if a.ndim > 2 else a for a in F]
    x, u, cost, _, st = O.lqr(*F)
    assert not st.any()
    out.update(x=x, u=u, cost=cost)
    f = {k: None if v is None else v.float() for k, v in ins.items()}
    ns, nc = meta["ns"], meta["nc"]
    lqr = pb.module.LQR(pb.module.LTI(f["A"], f["B"], torch.eye(ns).expand(nb, ns, ns), torch.zeros(nb, ns, nc), f["c1"]),
                        f["Q"], f["p"], T)
    K, k = lqr.lqr_backward(f["x0"], 1, f["u_traj"])
    meta["err32"] = err32(lqr.lqr_forward(f["x0"], K, k), out)
    meta["systime"] = 2 * T - 1
    return meta, out


class CartPole(pp.module.NLS):
    """the standard cart-pole: state (x, x', theta, theta'), input the force, explicit Euler step of length dt"""

    def __init__(self, dt=0.01, length=1.5, cartmass=20.0, polemass=10.0, gravity=9.81):
        super().__init__()
        self.tau, self.length, self.polemass, self.gravity = dt, length, polemass, gravity
        self.poleml, self.total = polemass * length, cartmass + polemass

    def state_transition(self, state, input, t=None):
        x, xd, th, thd = state.squeeze()
        force = input.squeeze()
        c, s = torch.cos(th), torch.sin(th)
        tmp = (force + self.poleml * thd ** 2 * s) / self.total
        thacc = (self.gravity * s - c * tmp) / (self.length * (4.0 / 3.0 - self.polemass * c ** 2 / self.total))
        xacc = tmp - self.poleml * thacc * c / self.total
        return (state.squeeze() + torch.stack((xd, xacc, thd, thacc)) * self.tau).unsqueeze(0)

    def observation(self, state, input, t=None):
        return state


def cartpole(mpc):
    g = torch.Generator().manual_seed(9)
    T, dt = 5, 0.01
    Q = torch.eye(5, dtype=D).repeat(1, T, 1, 1)
    p = torch.randn(1, T, 5, generator=g, dtype=D)
    x0 = torch.tensor([[0.0, 0.0, torch.pi, 0.0]], dtype=D)
    u0 = torch.sin(torch.arange(T, dtype=D) * dt).reshape(1, T, 1)
    if mpc:
        x, u, cost = pp.module.MPC(CartPole(dt), Q, p, T, stepper=pp.utils.ReduceToBason(10))(dt, x0, u_init=u0)
    else:
        x, u, cost = pp.module.LQR(CartPole(dt), Q, p, T)(x0, dt, u0)
    meta = dict(kind="nls_mpc" if mpc else "nls_lqr", nb=1, T=T, ns=4, nc=1, dt=dt, ltv=False, grad=False, raises=False,
                **{"from": "reference"})
    return meta, dict(Q=Q.numpy(), p=p.numpy(), x0=x0.numpy(), u_traj=u0.numpy(), x=x.detach().numpy(),
                      u=u.detach().numpy(), cost=cost.detach().numpy())


CASES = {
    "lti_2_5_4_3": dict(seed=1, nb=2, T=5, ns=4, nc=3, u=True, grad=True),
    "lti_16_50_6_2_shared": dict(seed=2, nb=16, T=50, ns=6, nc=2, q_step=False, p3=False, grad=True),
    "lti_64_20_12_4_shared_q": dict(seed=3, nb=64, T=20, ns=12, nc=4, q_step=False, c1=False),
    "lti_4_30_31_1_shared_q": dict(seed=5, nb=4, T=30, ns=31, nc=1, q_step=False, u=True),
    "ltv_3_8_5_2": dict(seed=6, nb=3, T=8, ns=5, nc=2, ltv=True, u=True, grad=True),
    "ltv_dt_half": dict(seed=7, nb=3, T=8, ns=5, nc=2, ltv=True, dt=0.5),
    "indefinite": dict(seed=8, nb=4, T=6, ns=3, nc=2, indefinite=True),
    "lti_8_10_1_1": dict(seed=4, nb=8, T=10, ns=1, nc=1),
}


def main():
    meta, arrays = {}, {}
    for name, kw in CASES.items():
        m, a = case(**kw)
        meta[name] = m
        arrays.update({f"{name}/{k}": v for k, v in a.items()})
    for name, mpc in (("cartpole_lqr", False), ("cartpole_mpc", True)):
        m, a = cartpole(mpc)
        meta[name] = m
        arrays.update({f"{name}/{k}": v for k, v in a.items()})
    np.savez_compressed(OUT, cases=json.dumps(meta), **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
