"""pp.module.LQR / MPC and the dynamics models (csrc/lqr.cu, csrc/lqr_math.cuh, module/lqr.py) against reference goldens
(oracle/make_golden_lqr.py) and the fp64 oracle (oracle/lqr_oracle.py).  DESIGN.md §3.7."""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import lqr_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "lqr.npz"))
CASES = json.loads(str(GOLD["cases"]))
SOLVED = [k for k, c in CASES.items() if not c["raises"] and c["kind"] in ("lti", "ltv")]
NLS = [k for k, c in CASES.items() if c["kind"].startswith("nls")]
GRAD = [k for k, c in CASES.items() if c["grad"]]
_HOST = {}


# ------------------------------------------------------------------ test-only CPU kernels of the new ops, from the oracle
def _np(t):
    return None if t is None else t.detach().double().cpu().numpy()


def _full(Q, p, A, B, c1, x_init, u_traj, T):
    nb = x_init.shape[0]
    Qf, pf, Af, Bf, cf, x0, uf = O.full(*(_np(t) for t in (Q, p, A, B, c1, x_init, u_traj)))
    b = lambda a: np.broadcast_to(a, (nb, T) + a.shape[2:])   # noqa: E731
    return b(Qf), b(pf), b(Af), b(Bf), b(cf), x0, b(uf)


def _cpu_fwd(Q, p, A, B, c1, x_init, u_traj, T):
    x, u, c, xt, st = O.lqr(*_full(Q, p, A, B, c1, x_init, u_traj, T))
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(x_init.dtype)   # noqa: E731
    return f(x), f(u), f(c), f(xt), torch.from_numpy(st)


def _cpu_bwd(Q, p, A, B, c1, x_init, T, x, u, gx, gu, gcost):
    F = _full(Q, p, A, B, c1, x_init, None, T)
    gs = O.lqr_bwd(*F[:6], _np(x), _np(u), _np(gx), _np(gu), _np(gcost))
    out = []
    for g, t in zip(gs[:5], (Q, p, A, B, c1)):
        if t is None:
            out.append(x_init.new_empty(0))
            continue
        if t.shape[1] == 1:
            g = g.sum(1, keepdims=True)
        out.append(torch.from_numpy(np.ascontiguousarray(g)).to(x_init.dtype))
    return (*out, torch.from_numpy(gs[5]).to(x_init.dtype))


torch.library.register_kernel("b200pose::lqr_affine", "cpu", _cpu_fwd)
torch.library.register_kernel("b200pose::lqr_affine_bwd", "cpu", _cpu_bwd)


class StepLTV(pp.module.LTV):
    """per-step A_t, B_t read at the system time (the goldens' time-varying system)"""
    @property
    def A(self):
        return self._A[:, int(self._t)]

    @property
    def B(self):
        return self._B[:, int(self._t)]


def golden(name, k):
    key = f"{name}/{k}"
    return GOLD[key] if key in GOLD.files else None


def inputs(name, device="cpu", dtype=torch.float64, grad=False):
    t = lambda k: None if golden(name, k) is None else \
        torch.tensor(golden(name, k), dtype=dtype, device=device).requires_grad_(grad)   # noqa: E731
    return {k: t(k) for k in ("Q", "p", "A", "B", "c1", "x0", "u_traj")}


def solve(name, ins, cls=None):
    c = CASES[name]
    ns, nc, nb = c["ns"], c["nc"], c["nb"]
    dev, dt = ins["x0"].device, ins["x0"].dtype
    C = torch.eye(ns, dtype=dt, device=dev).expand(nb, ns, ns)
    D = torch.zeros(nb, ns, nc, dtype=dt, device=dev)
    cls = cls or (StepLTV if c["ltv"] else pp.module.LTI)
    sys_ = cls(ins["A"], ins["B"], C, D, ins["c1"], None)
    lqr = pp.module.LQR(sys_, ins["Q"], ins["p"], c["T"])
    return lqr, sys_, lqr(ins["x0"], c["dt"], ins["u_traj"])


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _vp(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="lqr_host_")
        so = os.path.join(d, "liblqrhost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "lqr_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def full_case(name):
    c = CASES[name]
    g = lambda k: golden(name, k)   # noqa: E731
    nb, T = c["nb"], c["T"]
    Q, p = g("Q"), g("p")
    Q = Q if Q.ndim == 4 else Q[:, None]
    p = p if p.ndim == 3 else p[:, None]
    A, B = (g(k) if c["ltv"] else g(k)[:, None] for k in ("A", "B"))
    c1 = None if g("c1") is None else g("c1")[:, None]
    return [np.ascontiguousarray(a) for a in _full_np(Q, p, A, B, c1, g("x0"), g("u_traj"), nb, T)]


def _full_np(Q, p, A, B, c1, x0, u, nb, T):
    F = O.full(Q, p, A, B, c1, x0, u)
    return [np.broadcast_to(a, (nb, T) + a.shape[2:]) if a.ndim > 2 else a for a in F]


# ------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", SOLVED)
def test_oracle_reproduces_reference(name):
    if CASES[name]["dt"] != 1:
        pytest.skip("dt != 1 reads A_t at int(t * dt): not an affine problem in t")
    x, u, c, _, st = O.lqr(*full_case(name))
    assert not st.any()
    assert rel(x, golden(name, "x")) < 1e-10 and rel(u, golden(name, "u")) < 1e-10 and rel(c, golden(name, "cost")) < 1e-10


@pytest.mark.parametrize("name", GRAD)
def test_oracle_adjoint_matches_reference_autograd(name):
    F = full_case(name)
    gs = O.lqr_bwd(*F[:6], golden(name, "x"), golden(name, "u"), golden(name, "gx"), golden(name, "gu"), golden(name, "gc"))
    check_grads(name, dict(zip(("Q", "p", "A", "B", "c1", "x0"), gs)), reduce=True)


def check_grads(name, got, reduce, tol=1e-9):
    """got: gradients per key; reduce: full-size oracle output to be summed to the golden's shape"""
    c = CASES[name]
    for k in ("Q", "p", "A", "B", "c1", "x0"):
        want = golden(name, f"g{k}")
        if want is None:
            continue
        g = np.asarray(got[k])
        if reduce and g.ndim == want.ndim + 1:
            g = g.sum(1)
        if k == "Q":           # only the symmetric part of dQ is determined by the problem
            want = 0.5 * (want + np.swapaxes(want, -1, -2))
            g = 0.5 * (g + np.swapaxes(g, -1, -2))
        assert rel(g, want) < tol, (k, rel(g, want))


def test_indefinite_raises_in_oracle():
    assert O.lqr(*_full_np(*[golden("indefinite", k)[:, None] if k in ("A", "B", "c1") else golden("indefinite", k)
                              for k in ("Q", "p", "A", "B", "c1", "x0")], None, 4, 6))[4][0] == 1


@pytest.mark.parametrize("name", [n for n in SOLVED if CASES[n]["dt"] == 1])
def test_host_build_matches_oracle(name):
    c = CASES[name]
    Q, p, A, B, c1, x0, u0 = full_case(name)
    nb, T, ns, nc = c["nb"], c["T"], c["ns"], c["nc"]
    x, u, cost, xt = np.empty((nb, T + 1, ns)), np.empty((nb, T, nc)), np.empty(nb), np.empty((nb, T, ns))
    st = np.empty(nb, np.int32)
    _host().lqr_host_solve(*[_vp(a) for a in (Q, p, A, B, c1, x0, u0)], ctypes.c_longlong(nb), T, ns, nc,
                           _vp(x), _vp(u), _vp(cost), _vp(xt), _vp(st))
    xo, uo, co, xto, _ = O.lqr(Q, p, A, B, c1, x0, u0)
    assert not st.any()
    assert rel(x, xo) < 1e-11 and rel(u, uo) < 1e-11 and rel(cost, co) < 1e-11 and rel(xt, xto) < 1e-12
    if c["grad"]:
        gx, gu, gc = golden(name, "gx"), golden(name, "gu"), golden(name, "gc")
        outs = [np.empty(a.shape) for a in (Q, p, A, B, c1, x0)]
        _host().lqr_host_adjoint(*[_vp(a) for a in (Q, p, A, B, c1, x0)], ctypes.c_longlong(nb), T, ns, nc, _vp(xo),
                                 _vp(uo), _vp(gx), _vp(gu), _vp(gc), *[_vp(a) for a in outs])
        want = O.lqr_bwd(Q, p, A, B, c1, x0, xo, uo, gx, gu, gc)
        for g, w in zip(outs, want):
            assert rel(g, w) < 1e-10


@pytest.mark.parametrize("name", [n for n in SOLVED if CASES[n]["dt"] == 1])
def test_host_build_fp32_within_4x_of_the_fp32_reference(name):
    c = CASES[name]
    F = [None if a is None else np.ascontiguousarray(a, np.float32) for a in full_case(name)]
    nb, T, ns, nc = c["nb"], c["T"], c["ns"], c["nc"]
    out = {"x": np.empty((nb, T + 1, ns), np.float32), "u": np.empty((nb, T, nc), np.float32),
           "cost": np.empty(nb, np.float32)}
    xt, st = np.empty((nb, T, ns), np.float32), np.empty(nb, np.int32)
    _host().lqr_host_solve_f32(*[_vp(a) for a in F], ctypes.c_longlong(nb), T, ns, nc, _vp(out["x"]), _vp(out["u"]),
                               _vp(out["cost"]), _vp(xt), _vp(st))
    assert not st.any()
    for k, v in out.items():
        assert rel(v, golden(name, k)) <= 4 * c["err32"][k], (k, rel(v, golden(name, k)), c["err32"][k])


def check_module(name, lqr, sys_, x, u, cost, tol=1e-10):
    assert rel(x.detach().cpu(), golden(name, "x")) < tol and rel(u.detach().cpu(), golden(name, "u")) < tol
    assert rel(cost.detach().cpu(), golden(name, "cost")) < tol
    assert int(sys_.systime) == CASES[name]["systime"]
    torch.testing.assert_close(sys_.state, x[:, -2].detach())
    torch.testing.assert_close(sys_.input, u[:, -1].detach())
    assert lqr.x_traj.shape == (CASES[name]["nb"], CASES[name]["T"], CASES[name]["ns"])


@pytest.mark.parametrize("name", SOLVED)
def test_module_on_cpu_takes_the_generic_route(name):
    ins = inputs(name)
    lqr, _, _ = solve(name, ins)
    assert lqr._route(ins["x0"], CASES[name]["dt"], ins["u_traj"]) is None
    lqr, sys_, (x, u, cost) = solve(name, ins)
    check_module(name, lqr, sys_, x, u, cost)


@pytest.mark.parametrize("name", [n for n in SOLVED if CASES[n]["dt"] == 1])
def test_affine_route_logic_on_cpu_kernels(name):
    """the affine route's Python side (operands, strides, systime / state / input left behind) on the oracle-backed
    test kernel"""
    c, ins = CASES[name], inputs(name)
    nb, ns, nc = c["nb"], c["ns"], c["nc"]
    C, D = torch.eye(ns, dtype=torch.float64).expand(nb, ns, ns), torch.zeros(nb, ns, nc, dtype=torch.float64)
    sys_ = (StepLTV if c["ltv"] else pp.module.LTI)(ins["A"], ins["B"], C, D, ins["c1"], None)
    lqr = pp.module.LQR(sys_, ins["Q"], ins["p"], c["T"])
    x, u, cost = lqr._affine(ins["x0"], 1, ins["u_traj"], 'gather' if c["ltv"] else 'lti')
    check_module(name, lqr, sys_, x, u, cost)


def test_routes_on_cpu():
    ins = inputs("lti_2_5_4_3")
    lqr, _, _ = solve("lti_2_5_4_3", ins)
    assert lqr._route(ins["x0"], 1, ins["u_traj"]) is None


@pytest.mark.parametrize("steps", [3, 1, 6])
def test_mis_sized_Q_or_p_raises_as_the_reference(steps):
    """Q / p with a step axis other than T: the reference raises in its recursion, and so does the generic route"""
    ins = inputs("lti_2_5_4_3")
    C, D = torch.eye(4, dtype=torch.float64).expand(2, 4, 4), torch.zeros(2, 4, 3, dtype=torch.float64)
    lti = pp.module.LTI(ins["A"], ins["B"], C, D, ins["c1"])
    Q, p = ins["Q"][:, :1].expand(2, steps, 7, 7).contiguous(), ins["p"][:, :1].expand(2, steps, 7).contiguous()
    lqr = pp.module.LQR(lti, Q, p, 5)
    assert lqr._route(ins["x0"], 1, None) is None
    with pytest.raises((RuntimeError, IndexError)):
        lqr(ins["x0"])


@pytest.mark.parametrize("name", ["lti_2_5_4_3", "ltv_3_8_5_2", "lti_16_50_6_2_shared"])
def test_generic_route_matches_goldens(name):
    ins = inputs(name)
    lqr, sys_, _ = solve(name, ins)
    sys_.reset()
    K, k = lqr.lqr_backward(ins["x0"], 1, ins["u_traj"])
    x, u, cost = lqr.lqr_forward(ins["x0"], K, k)
    assert rel(x, golden(name, "x")) < 1e-10 and rel(u, golden(name, "u")) < 1e-10


@pytest.mark.parametrize("name", GRAD)
def test_module_grads_on_cpu_kernels(name):
    ins = inputs(name, grad=True)
    _, _, (x, u, cost) = solve(name, ins)
    gx, gu, gc = (torch.tensor(golden(name, k)) for k in ("gx", "gu", "gc"))
    keys = [k for k in ("Q", "p", "A", "B", "c1", "x0") if ins[k] is not None]
    gr = torch.autograd.grad((x * gx).sum() + (u * gu).sum() + (cost * gc).sum(), [ins[k] for k in keys])
    check_grads(name, dict(zip(keys, gr)), reduce=False)


@pytest.mark.parametrize("name", GRAD)
def test_affine_grads_on_cpu_kernels(name):
    c, ins = CASES[name], inputs(name, grad=True)
    nb, ns, nc = c["nb"], c["ns"], c["nc"]
    C, D = torch.eye(ns, dtype=torch.float64).expand(nb, ns, ns), torch.zeros(nb, ns, nc, dtype=torch.float64)
    lqr = pp.module.LQR((StepLTV if c["ltv"] else pp.module.LTI)(ins["A"], ins["B"], C, D, ins["c1"], None),
                        ins["Q"], ins["p"], c["T"])
    x, u, cost = lqr._affine(ins["x0"], 1, ins["u_traj"], 'gather' if c["ltv"] else 'lti')
    gx, gu, gc = (torch.tensor(golden(name, k)) for k in ("gx", "gu", "gc"))
    keys = [k for k in ("Q", "p", "A", "B", "c1", "x0") if ins[k] is not None]
    gr = torch.autograd.grad((x * gx).sum() + (u * gu).sum() + (cost * gc).sum(), [ins[k] for k in keys])
    check_grads(name, dict(zip(keys, gr)), reduce=False)


def test_indefinite_raises():
    with pytest.raises(torch.linalg.LinAlgError):
        solve("indefinite", inputs("indefinite"))


def test_mpc_linear_system_equals_lqr():
    ins = inputs("lti_2_5_4_3")
    ins["x0"] = ins["x0"][:1]
    ins = {k: (v[:1] if v is not None else None) for k, v in ins.items()}
    C = torch.eye(4, dtype=torch.float64).expand(1, 4, 4)
    D = torch.zeros(1, 4, 3, dtype=torch.float64)
    lti = pp.module.LTI(ins["A"], ins["B"], C, D, ins["c1"], None)
    x, u, cost = pp.module.MPC(lti, ins["Q"], ins["p"], 5, stepper=pp.utils.ReduceToBason(4))(1, ins["x0"])
    xo, uo, co, _, _ = O.lqr(*_full_np(ins["Q"].numpy(), ins["p"].numpy(), ins["A"].numpy()[:, None],
                                       ins["B"].numpy()[:, None], ins["c1"].numpy()[:, None], ins["x0"].numpy(), None, 1, 5))
    assert rel(x, xo) < 1e-10 and rel(cost, co) < 1e-10


def test_mpc_without_iterations_solves_from_u_init():
    ins = {k: (v[:1] if v is not None else None) for k, v in inputs("lti_2_5_4_3").items()}
    C, D = torch.eye(4, dtype=torch.float64).expand(1, 4, 4), torch.zeros(1, 4, 3, dtype=torch.float64)
    class Stopped(pp.utils.ReduceToBason):            # a stepper that ends the loop before its first pass
        def continual(self):
            return False
    mpc = pp.module.MPC(pp.module.LTI(ins["A"], ins["B"], C, D, ins["c1"]), ins["Q"], ins["p"], 5,
                        stepper=Stopped(3))
    mpc(1, ins["x0"], u_init=ins["u_traj"])
    assert mpc.lqr.u_traj is ins["u_traj"]


class CartPole(pp.module.NLS):
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


def cartpole(name, device):
    c = CASES[name]
    Q, p, x0, u0 = (torch.tensor(golden(name, k), device=device) for k in ("Q", "p", "x0", "u_traj"))
    dt, T = c["dt"], c["T"]
    if c["kind"] == "nls_mpc":
        mpc = pp.module.MPC(CartPole(dt).to(device), Q, p, T, stepper=pp.utils.ReduceToBason(10))
        assert mpc.lqr._route(x0, dt, u0) is None
        return mpc(dt, x0, u_init=u0)
    return pp.module.LQR(CartPole(dt).to(device), Q, p, T)(x0, dt, u0)


@pytest.mark.parametrize("name", NLS)
def test_cartpole_generic_route_matches_goldens(name):
    x, u, cost = cartpole(name, "cpu")
    assert rel(x, golden(name, "x")) < 1e-10 and rel(u, golden(name, "u")) < 1e-10
    assert rel(cost, golden(name, "cost")) < 1e-10


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name", SOLVED)
def test_gpu_matches_goldens(name, dtype):
    """fp64: 1e-10 relative; fp32: within 4x the fp32 reference's own error against the fp64 goldens"""
    lqr, sys_, (x, u, cost) = solve(name, inputs(name, "cuda", dtype))
    for got, k in ((x, "x"), (u, "u"), (cost, "cost")):
        tol = 1e-10 if dtype == torch.float64 else 4 * CASES[name]["err32"][k]
        assert rel(got.cpu(), golden(name, k)) <= tol, (k, rel(got.cpu(), golden(name, k)), tol)
    assert int(sys_.systime) == CASES[name]["systime"]


@pytest.mark.gpu
def test_gpu_routes():
    ins = inputs("lti_2_5_4_3", "cuda")
    lqr, _, _ = solve("lti_2_5_4_3", ins)
    assert lqr._route(ins["x0"], 1, ins["u_traj"]) == 'lti'
    ins = inputs("ltv_3_8_5_2", "cuda")
    lqr, _, _ = solve("ltv_3_8_5_2", ins)
    lqr.system.reset()
    assert lqr._route(ins["x0"], 1, None) == 'gather'
    assert lqr._route(ins["x0"], 0.5, None) is None
    lqr.system.reset(1)
    assert lqr._route(ins["x0"], 1, None) is None

    class MyLTI(pp.module.LTI):                       # a user transition
        def state_transition(self, state, input):
            return super().state_transition(state, input)

    class PropLTI(pp.module.LTI):                     # an LTI with a property: the reference reads it at other times
        @property
        def A(self):
            return self._A

    ins = inputs("lti_2_5_4_3", "cuda")
    for cls in (MyLTI, PropLTI):
        lqr, sys_, (x, u, cost) = solve("lti_2_5_4_3", ins, cls=cls)
        assert lqr._route(ins["x0"], 1, None) is None
        check_module("lti_2_5_4_3", lqr, sys_, x, u, cost)
    lqr, _, _ = solve("lti_2_5_4_3", ins)
    lqr.p = lqr.p[:, :3]
    lqr.Q = lqr.Q[:, :3]
    assert lqr._route(ins["x0"], 1, None) is None
    with pytest.raises((RuntimeError, IndexError)):
        lqr(ins["x0"])


@pytest.mark.gpu
def test_gpu_op_rejects_mis_sized_or_mismatched_operands():
    ins = inputs("lti_2_5_4_3", "cuda")
    A, B, c1 = ins["A"][:, None], ins["B"][:, None], ins["c1"][:, None]
    with pytest.raises(ValueError):
        torch.ops.b200pose.lqr_affine(ins["Q"].cpu(), ins["p"], A, B, c1, ins["x0"], None, 5)
    with pytest.raises(ValueError):
        torch.ops.b200pose.lqr_affine(ins["Q"][:, :3], ins["p"], A, B, c1, ins["x0"], None, 5)
    with pytest.raises(ValueError):
        torch.ops.b200pose.lqr_affine(ins["Q"], ins["p"], A, B, c1, ins["x0"], None, 6)
    with pytest.raises(ValueError):
        torch.ops.b200pose.lqr_affine(ins["Q"], ins["p"], A.float(), B, c1, ins["x0"], None, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NLS)
def test_gpu_cartpole_generic_route_matches_goldens(name):
    x, u, cost = cartpole(name, "cuda")
    assert rel(x.cpu(), golden(name, "x")) < 1e-10 and rel(u.cpu(), golden(name, "u")) < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize("name", GRAD)
def test_gpu_grads_match_reference_autograd(name):
    ins = inputs(name, "cuda", grad=True)
    _, _, (x, u, cost) = solve(name, ins)
    gx, gu, gc = (torch.tensor(golden(name, k), device="cuda") for k in ("gx", "gu", "gc"))
    keys = [k for k in ("Q", "p", "A", "B", "c1", "x0") if ins[k] is not None]
    gr = torch.autograd.grad((x * gx).sum() + (u * gu).sum() + (cost * gc).sum(), [ins[k] for k in keys])
    check_grads(name, {k: g.cpu().numpy() for k, g in zip(keys, gr)}, reduce=False)


def _small(dev, dtype=torch.float64, nb=2, T=4, ns=3, nc=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = ns + nc
    M = torch.randn(nb, T, n, n, generator=g, dtype=dtype)
    Q = M.mT @ M + torch.eye(n, dtype=dtype)
    r = lambda *s: torch.randn(*s, generator=g, dtype=dtype)   # noqa: E731
    ops = (Q, r(nb, T, n), 0.8 * torch.eye(ns, dtype=dtype) + 0.2 / ns ** 0.5 * r(nb, 1, ns, ns), r(nb, 1, ns, nc), r(nb, 1, ns),
           r(nb, ns), r(nb, T, nc))
    return [t.to(dev) for t in ops]


@pytest.mark.gpu
def test_gpu_gradcheck_and_opcheck():
    Q, p, A, B, c1, x0, ut = _small("cuda")
    args = [t.requires_grad_() for t in (Q, p, A, B, c1, x0)]

    def f(Q, p, A, B, c1, x0):
        x, u, c, _, _ = torch.ops.b200pose.lqr_affine(0.5 * (Q + Q.mT), p, A, B, c1, x0, ut, 4)
        return x, u, c
    assert torch.autograd.gradcheck(f, args, atol=1e-7, rtol=1e-6)
    torch.library.opcheck(torch.ops.b200pose.lqr_affine, (Q.detach(), p.detach(), A.detach(), B.detach(), c1.detach(),
                                                          x0.detach(), ut, 4))


@pytest.mark.gpu
def test_gpu_stride0_equals_materialised():
    Q, p, A, B, c1, x0, _ = _small("cuda", nb=8, T=16, ns=6, nc=3)
    Q1, p1 = Q[:1, :1], p[:, :1]
    a = torch.ops.b200pose.lqr_affine(Q1, p1, A, B, c1, x0, None, 16)
    b = torch.ops.b200pose.lqr_affine(Q1.expand(8, 16, 9, 9).contiguous(), p1.expand(8, 16, 9).contiguous(),
                                      A.expand(8, 16, 6, 6).contiguous(), B.expand(8, 16, 6, 3).contiguous(),
                                      c1.expand(8, 16, 6).contiguous(), x0, torch.zeros(8, 16, 3, device="cuda", dtype=Q.dtype), 16)
    for s, t in zip(a[:4], b[:4]):
        assert torch.equal(s, t)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_gpu_large_batch_against_oracle(dtype):
    nb, T, ns, nc = 20000, 64, 6, 2
    Q, p, A, B, c1, x0, ut = _small("cpu", torch.float64, nb=nb, T=1, ns=ns, nc=nc, seed=3)
    pT = torch.randn(nb, T, ns + nc, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
    dev = [t.to("cuda", dtype) for t in (Q, pT, A, B, c1, x0)]
    x, u, cost, _, st = torch.ops.b200pose.lqr_affine(*dev, None, T)
    assert not st.any()
    idx = np.random.default_rng(0).choice(nb, 32, replace=False)
    want = O.lqr(*_full_np(Q.numpy()[idx], pT.numpy()[idx], A.numpy()[idx], B.numpy()[idx], c1.numpy()[idx],
                           x0.numpy()[idx], None, 32, T))
    if dtype == torch.float64:
        assert rel(x.cpu()[idx], want[0]) < 1e-10 and rel(cost.cpu()[idx], want[2]) < 1e-10
        return
    # fp32: within 4x the error of the reference's algorithm run in fp32 (the generic route, on the CPU) on the sample
    f = lambda t: t[idx].float()   # noqa: E731
    lti = pp.module.LTI(f(A)[:, 0], f(B)[:, 0], torch.eye(ns).expand(32, ns, ns), torch.zeros(32, ns, nc), f(c1)[:, 0])
    lqr = pp.module.LQR(lti, f(Q)[:, 0], f(pT), T)
    K, k = lqr.lqr_backward(f(x0), 1)
    xr, _, cr = lqr.lqr_forward(f(x0), K, k)
    assert rel(x.cpu()[idx], want[0]) <= 4 * rel(xr, want[0]) and rel(cost.cpu()[idx], want[2]) <= 4 * rel(cr, want[2])


@pytest.mark.gpu
def test_gpu_one_indefinite_problem_in_a_large_batch_raises():
    nb, T, ns, nc = 5000, 8, 4, 2
    Q, p, A, B, c1, x0, _ = _small("cpu", nb=nb, T=T, ns=ns, nc=nc, seed=5)
    Q[1234, 3, ns:, ns:] -= 1e3 * torch.eye(nc, dtype=Q.dtype)
    C, D = torch.eye(ns, dtype=Q.dtype).expand(nb, ns, ns), torch.zeros(nb, ns, nc, dtype=Q.dtype)
    lti = pp.module.LTI(A[:, 0].cuda(), B[:, 0].cuda(), C.cuda(), D.cuda(), c1[:, 0].cuda())
    with pytest.raises(torch.linalg.LinAlgError):
        pp.module.LQR(lti, Q.cuda(), p.cuda(), T)(x0.cuda())


@pytest.mark.gpu
def test_gpu_generic_route_matches_goldens():
    name = "ltv_dt_half"
    _, _, (x, u, cost) = solve(name, inputs(name, "cuda"))
    assert rel(x.cpu(), golden(name, "x")) < 1e-10 and rel(cost.cpu(), golden(name, "cost")) < 1e-10
