"""Gradients of the LieTensor API through the CUDA kernels: the torch.autograd.Functions and vmap rules of
pypose_b200/lietensor/ops.py (and Jinvp's group gradient, _jinvp_composite.py) against two fp64 references.

1. The same Python function on CPU fp64 copies of the inputs.  On CPU every b200pose op runs the oracle
   (tests/conftest.py), so this is an fp64 evaluation of the exact autograd graph.  It runs under
   `lie_oracle.wide_taylor()`: the reference's formulas evaluated without their own small-angle cancellation.
2. Central differences of the oracle's forward in numpy (fourth-order stencil, h = 3e-4), independent of the wiring.
   Algebra and plain-tensor inputs are perturbed componentwise; group inputs on the left, X <- Exp(delta) X, and
   their last D - K gradient entries must be exactly 0.  Ops with a group output are differentiated through
   phi(Z) = w . Log(Z Z0^-1), whose left-tangent gradient at Z0 is exactly [w, 0], so the cotangent [w, 0] is
   what autograd is given.  The differences use `wide_taylor()` too: the reference-faithful forward evaluates
   closed forms such as calcQ's c2 = (theta^2 + 2 cos(theta) - 2) / (2 theta^4) down to theta = machine eps, where
   the rounding of cos(theta) leaves ~1e-11 of noise at theta = 1e-4; divided by 2h = 2e-6 that alone is 5e-6.

Sim3's Exp and Log backward use the reference's truncated series for Jl and Jl^-1 (oracle/lie_oracle.py
sim3_Jl / sim3_Jl_inv, "approximate by design"), so Sim3 Exp (and Retr's algebra operand), Log and Jinvp(X) are held
to the gradient the reference defines instead: g @ sim3_Jl(x), g @ sim3_Jl_inv(x), and for Jinvp the Euclidean
derivative of x -> w . sim3_Jl_inv(x) p chained through g @ sim3_Jl_inv(x).  The truncation is ~5e-3 at |x| ~ 1.

SE3 Jinvp's group gradient: the composite computes d/dx[Jl^-1(x) p] (closed-form Jl^-1 and Q, series below
theta^2 = 1e-4) chained through Log's backward g @ Jl^-1(x).  The reference has no custom backward either: autograd
through SE3_Log.backward (g @ se3_Jl_inv(x)) and the explicit calcQ matrix build, i.e. the same derivative.  It
matches the left-tangent differences of the exact forward to the differences' own error (test_jinvp_group_gradient).
Second-order differences with h = 1e-6 of the reference-faithful forward disagree with it by up to 7e-6; that is the
forward's rounding noise (the c2 cancellation above, and eps |f| / h with |tau| ~ 5), not a gradient error: it
vanishes with wide_taylor().  What the tests found wrong was fp32: the composite ran in the input dtype, and in fp32 its
closed-form c2 / c3 have no correct digits for theta in (0.01, 0.03), which gave gX errors of 2e-2 at theta = 0.0101.
It now runs in fp64 for every dtype.

Rows: rotation angles {1e-6, 1e-3, 0.01 (1 -+ 1e-3) on both sides of the series switch, pi - 1e-3} on random axes,
random angles in (0.05, pi - 0.05), RxSO3 / Sim3 log-scales +-3 (scales e^+-3) among N(0, 0.5) ones, and w < 0
quaternions on every other group row.

Bounds.  fp64 is judged relative to (1 + |truth|), fp32 relative to (term_scale x (1 + |w|) + |truth|) (tests/util.py;
the cotangent w multiplies every gradient term).  Measured maxima on an H100 SXM (CPU for the cpu rows):
  * reference 1, forward and gradients of every op and group: fp64 1.5e-12 (SE3 Jinvp dX), fp32 8.1e-8.
  * chains: fp64 1.1e-12, fp32 7.0e-8; Exp->Log at 10^6 rows, fp32: 4.0e-7.  Broadcasting: fp64 4.6e-15, fp32 6.2e-8.
  * finite differences: fp64 4.7e-9 (cpu and H100 alike), fp32 1.4e-7.  Jinvp's group gradient: 2.4e-8 (SE3, |tau| ~ 5).
"""
import os
import zlib

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import lie_oracle as O
from pypose_b200._optable import GROUPS
from tests.util import QUAT_SLICE, ROT_SLICE, term_scale

GPU = pytest.mark.gpu
F64, F32 = torch.float64, torch.float32
TYPES = {"SO3": (pp.SO3_type, pp.so3_type), "SE3": (pp.SE3_type, pp.se3_type),
         "RxSO3": (pp.RxSO3_type, pp.rxso3_type), "Sim3": (pp.Sim3_type, pp.sim3_type)}
# fp64: the kernels' 1e-12 of test_lie_gpu.py, with room for the roundings of a chain of kernels and of Jinvp's composite
# (torch matrix products between two kernels).  fp32: the 1e-6 forward-error bound of test_lie_gpu.py.
TOL = {F64: 5e-12, F32: 1e-6}
# fp64 against finite differences: the stencil's own error.  Its h^4 truncation is below 1e-12 here; what remains is the
# oracle's rounding divided by h, largest just above wide_taylor's switch at theta = 1e-2, where the closed-form
# c2 = (theta^2 + 2 cos(theta) - 2) / (2 theta^4) keeps ~1e-16 / (theta^4 / 6) = 7e-8 of relative noise: ~3e-12 on a
# forward of size 10, 2e-8 in the difference.
TOL_FD = {F64: 1e-7, F32: 1e-6}
EDGE_THETA = (1e-6, 1e-3, 0.01 * (1 - 1e-3), 0.01 * (1 + 1e-3), np.pi - 1e-3)


def _dev_params(cpu=True):
    out = [pytest.param("cpu", F64, id="cpu-f64")] if cpu else []
    return out + [pytest.param("cuda", F64, id="f64", marks=GPU), pytest.param("cuda", F32, id="f32", marks=GPU)]


def _lt(t, grp, algebra=False):
    return pp.LieTensor(t, ltype=TYPES[grp][1 if algebra else 0])


def _raw(t):
    return t.tensor() if isinstance(t, pp.LieTensor) else t


# ---------------------------------------------------------------------------------------------------------------------
# ops: (input kinds, the LieTensor call, the oracle forward, output kind).  Kinds: G group, A algebra, T tangent vector,
# P3 / P4 points.  Output kinds: G group (cotangent [w, 0], differences through Log(Z Z0^-1)), V vector.
# ---------------------------------------------------------------------------------------------------------------------
OPS = {
    "Exp": (("A",), lambda g, x: _lt(x, g, True).Exp(), lambda g, x: O.exp(g, x), "G"),
    "Log": (("G",), lambda g, X: _lt(X, g).Log(), lambda g, X: O.log(g, X), "V"),
    "Inv": (("G",), lambda g, X: _lt(X, g).Inv(), lambda g, X: O.inv(g, X), "G"),
    "Mul": (("G", "G"), lambda g, X, Y: _lt(X, g) @ _lt(Y, g), lambda g, X, Y: O.mul(g, X, Y), "G"),
    "Act": (("G", "P3"), lambda g, X, p: _lt(X, g).Act(p), lambda g, X, p: O.act(g, X, p), "V"),
    "Act4": (("G", "P4"), lambda g, X, p: _lt(X, g).Act(p), lambda g, X, p: O.act4(g, X, p), "V"),
    "Adj": (("G", "T"), lambda g, X, a: _lt(X, g).Adj(_lt(a, g, True)), lambda g, X, a: O.adj(g, X, a), "V"),
    "AdjT": (("G", "T"), lambda g, X, a: _lt(X, g).AdjT(_lt(a, g, True)), lambda g, X, a: O.adjt(g, X, a), "V"),
    "Jinvp": (("G", "T"), lambda g, X, p: _lt(X, g).Jinvp(p), lambda g, X, p: O.jinvp(g, X, p), "V"),
    "Retr": (("G", "A"), lambda g, X, a: _lt(X, g).Retr(_lt(a, g, True)),
             lambda g, X, a: O.mul(g, O.exp(g, a), X), "G"),
}
# The reference's AdjT backward (operation.py SE3_AdjTXa / Sim3_AdjTXa) is the derivative of Adj(X)^T a, while its
# forward is Adj(X^-1) a; the two agree where Adj(X) is orthogonal (SO3, RxSO3).  For SE3 and Sim3 the differences are
# taken of the function the backward differentiates (module docstring).
FD_FWD = {("SE3", "AdjT"): lambda g, X, a: O._rowmat(a, O.ADJ[g](X)),
          ("Sim3", "AdjT"): lambda g, X, a: O._rowmat(a, O.ADJ[g](X))}
# (group, op, input) whose reference gradient is the truncated Sim3 series (module docstring)
SERIES = {("Sim3", "Exp", 0), ("Sim3", "Retr", 1), ("Sim3", "Log", 0), ("Sim3", "Jinvp", 0)}


def edge_algebra(rng, grp, n_rand=12, thetas=EDGE_THETA, per=4, t_sigma=1.0):
    """algebra rows: `per` random axes at each angle of `thetas`, then `n_rand` angles in (0.05, pi - 0.05);
    translations N(0, t_sigma); log-scales N(0, 0.5) with every third row at +-3"""
    K = GROUPS[grp][2]
    th = np.concatenate([np.repeat(np.asarray(thetas, float), per), rng.uniform(0.05, np.pi - 0.05, n_rand)])
    n = th.size
    x = rng.standard_normal((n, K)) * t_sigma
    d = rng.standard_normal((n, 3))
    x[:, ROT_SLICE[grp]] = d / np.linalg.norm(d, axis=1, keepdims=True) * th[:, None]
    if grp in ("RxSO3", "Sim3"):
        x[:, -1] = rng.standard_normal(n) * 0.5
        x[::3, -1] = np.where(rng.random(n)[::3] < 0.5, -3.0, 3.0)
    return x


def edge_group(rng, grp, **kw):
    X = O.exp(grp, edge_algebra(rng, grp, **kw))
    X[1::2, QUAT_SLICE[grp]] *= -1                 # w < 0 quaternions: the same group elements
    return X


def make_inputs(grp, op, seed=0):
    rng = np.random.default_rng(zlib.crc32(f"{grp}/{op}/{seed}".encode()))
    K = GROUPS[grp][2]
    ins = []
    for kind in OPS[op][0]:
        if kind == "G":
            ins.append(edge_group(rng, grp))
        elif kind == "A":
            ins.append(edge_algebra(rng, grp))
        else:
            ins.append(rng.standard_normal((ins[0].shape[0] if ins else 32, {"T": K, "P3": 3, "P4": 4}[kind])))
    n = min(a.shape[0] for a in ins)
    return [a[:n] for a in ins]


def _np(t):
    return t.detach().double().cpu().numpy()


def _report(what, err):
    if os.environ.get("B200POSE_REPORT_ERR"):       # dev: collect the measured maxima quoted in the docstring
        with open(os.environ["B200POSE_REPORT_ERR"], "a") as f:
            f.write(f"ERR {what} max={err:.3e}\n")


def check(res, truth, tol, what, scale=1.0):
    res, truth = np.asarray(res, np.float64), np.asarray(truth, np.float64)
    assert res.shape == truth.shape, (what, res.shape, truth.shape)
    assert np.isfinite(res).all(), what
    err = np.abs(res - truth) / (scale + np.abs(truth))
    e = float(err.max()) if err.size else 0.0
    _report(what, e)
    assert e <= tol, f"{what}: max rel err {e:.3e} > {tol:.0e}"


def fp32_scale(grp, op, ins, w):
    """term_scale of the op's inputs times (1 + |w|): every gradient term carries one factor of the cotangent"""
    return term_scale(grp, f"{op.lower()}_fwd", ins) * (1 + np.abs(w).max(1, keepdims=True))


def run_graph(fn, ins, cot, dev, dtype, wide=False):
    """(output, gradients) of sum(cot * fn(*ins)) with the inputs as leaves on `dev` in `dtype`"""
    ts = [torch.from_numpy(np.ascontiguousarray(a)).to(dev, dtype).requires_grad_() for a in ins]
    if wide:
        with O.wide_taylor():
            out = _raw(fn(*ts))
            grads = torch.autograd.grad(out, ts, torch.from_numpy(cot).to(dev, dtype))
    else:
        out = _raw(fn(*ts))
        grads = torch.autograd.grad(out, ts, torch.from_numpy(cot).to(dev, dtype))
    return out, grads, ts


# ---------------------------------------------------------------------------------------------------------------------
# finite differences (reference 2)
# ---------------------------------------------------------------------------------------------------------------------
H = 3e-4                    # 2H stays inside the pi - 1e-3 rows: no stencil crosses Log's cut at theta = pi


def _stencil(f, perturb, K):
    """fourth-order central difference of the per-row scalar f(perturb(delta)) in each of K directions"""
    n = None
    cols = []
    for k in range(K):
        vals = []
        for s in (1, -1, 2, -2):
            vals.append(f(perturb(k, s * H)))
        n = vals[0].shape[0]
        cols.append((8 * (vals[0] - vals[1]) - (vals[2] - vals[3])) / (12 * H))
    return np.stack(cols, 1) if cols else np.zeros((n or 0, 0))


def fd_gradients(grp, op, ins, w):
    """per input: the left-tangent (group) or Euclidean gradient of the per-row w . F, F the oracle forward (or
    w . Log(Z Z0^-1) for a group output), in wide_taylor mode"""
    kinds, _, fwd, out_kind = OPS[op]
    fwd = FD_FWD.get((grp, op), fwd)
    D, K = GROUPS[grp][1], GROUPS[grp][2]
    with O.wide_taylor():
        Z0i = O.inv(grp, fwd(grp, *ins)) if out_kind == "G" else None

        def phi(args):
            out = fwd(grp, *args)
            if out_kind == "G":
                out = O.log(grp, O.mul(grp, out, Z0i))
            return (w[:, :out.shape[1]] * out).sum(1)

        grads = []
        for i, kind in enumerate(kinds):
            def perturb(k, h, i=i, kind=kind):
                args = list(ins)
                if kind == "G":
                    d = np.zeros((ins[i].shape[0], K))
                    d[:, k] = h
                    args[i] = O.mul(grp, O.exp(grp, d), ins[i])
                else:
                    a = ins[i].copy()
                    a[:, k] += h
                    args[i] = a
                return args
            grads.append(_stencil(phi, perturb, K if kind == "G" else ins[i].shape[1]))
    return grads


def series_gradient(op, i, ins, w):
    """the gradient the reference defines through Sim3's truncated Jl / Jl^-1 (module docstring)"""
    K = 7
    wk = w[:, :K]
    with O.wide_taylor():
        if op in ("Exp", "Retr"):
            return O.exp_bwd("Sim3", ins[i], O._pad0(wk))
        x = O.log("Sim3", ins[0])
        if op == "Log":
            return O.log_bwd("Sim3", x, wk)[:, :K]
        # Jinvp: Euclidean derivative of x -> w . sim3_Jl_inv(x) p, chained through Log's backward
        p = ins[1]
        f = lambda xx: (wk * O._matvec(O.sim3_Jl_inv(xx), p)).sum(1)

        def perturb(k, h):
            a = x.copy()
            a[:, k] += h
            return a
        gx = _stencil(f, perturb, K)
        return O.log_bwd("Sim3", x, gx)[:, :K]


def _cotangent(grp, op, ins, seed):
    rng = np.random.default_rng(seed)
    kinds, _, fwd, out_kind = OPS[op]
    with O.wide_taylor():
        width = fwd(grp, *ins).shape[1]
    return rng.standard_normal((ins[0].shape[0], width))


@pytest.mark.parametrize("dev,dtype", _dev_params())
@pytest.mark.parametrize("grp", list(GROUPS))
@pytest.mark.parametrize("op", list(OPS))
def test_op_gradients_match_finite_differences(op, grp, dev, dtype):
    D, K = GROUPS[grp][1], GROUPS[grp][2]
    kinds, call, fwd, out_kind = OPS[op]
    ins = make_inputs(grp, op)
    ins = [np.asarray(torch.from_numpy(a).to(dtype).double()) for a in ins]     # the differences see the rounded rows
    w = _cotangent(grp, op, ins, 1)
    cot = w.copy()
    if out_kind == "G":
        cot[:, K:] = 0
    _, grads, _ = run_graph(lambda *t: call(grp, *t), ins, cot, dev, dtype)
    fd = fd_gradients(grp, op, ins, cot)
    for i, (kind, g) in enumerate(zip(kinds, grads)):
        g = _np(g)
        what = f"FD {dev}-{dtype} {grp} {op} d{i}"
        if kind == "G":
            assert (g[:, K:] == 0).all(), f"{what}: last D-K gradient entries not 0"
            g = g[:, :K]
        truth = series_gradient(op, i, ins, cot) if (grp, op, i) in SERIES else fd[i]
        scale = 1.0 if dtype == F64 else fp32_scale(grp, op, ins, w)
        check(g, truth, TOL_FD[dtype], what, scale)


# ---------------------------------------------------------------------------------------------------------------------
# the same graph in fp64 on CPU (reference 1)
# ---------------------------------------------------------------------------------------------------------------------
def compare_with_cpu_graph(fn, ins, cot, dtype, what, grp=None, op=None, scale_ins=None):
    out, grads, ts = run_graph(fn, ins, cot, "cuda", dtype)
    assert out.dtype == dtype and all(g.dtype == dtype and g.shape == t.shape for g, t in zip(grads, ts))
    host = [_np(t) for t in ts]                                 # fp64 copies of the rounded inputs
    out_h, grads_h, _ = run_graph(fn, host, _np(torch.from_numpy(cot).to(dtype)), "cpu", F64, wide=True)
    if dtype == F64:
        scale_o = scale_g = 1.0
    else:
        # one scalar: the product over the inputs of their largest row term (operands may be broadcast)
        s = np.prod([term_scale(grp, f"{op.lower()}_fwd", [h.reshape(-1, h.shape[-1])]).max()
                     for h in (scale_ins or host)])
        scale_o, scale_g = s, s * (1 + np.abs(cot).max())
    check(_np(out), _np(out_h), TOL[dtype], f"{what} out", scale_o)
    for i, (g, gh) in enumerate(zip(grads, grads_h)):
        check(_np(g), _np(gh), TOL[dtype], f"{what} d{i}", scale_g)
    return grads


@GPU
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("grp", list(GROUPS))
@pytest.mark.parametrize("op", list(OPS))
def test_op_forward_and_gradients_match_cpu_fp64_graph(op, grp, dtype):
    """every op, every group, with a random cotangent on every output entry (the group ones' last D - K included)"""
    ins = make_inputs(grp, op, seed=1)
    cot = _cotangent(grp, op, ins, 2)
    compare_with_cpu_graph(lambda *t: OPS[op][1](grp, *t), ins, cot, dtype, f"ref1 {grp} {op} {dtype}", grp, op)


CHAINS = {
    # name: (input kinds, function, op whose term_scale bounds the fp32 terms)
    "YExpLog": (("G", "A"), lambda g, Y, x: (_lt(Y, g) @ _lt(x, g, True).Exp()).Log(), "mul"),
    "InvMul": (("G", "G"), lambda g, X, Y: _lt(X, g).Inv() @ _lt(Y, g), "mul"),
    "MulAct": (("G", "G", "P3"), lambda g, X, Y, p: (_lt(X, g) @ _lt(Y, g)).Act(p), "mul"),
}


@GPU
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("grp", list(GROUPS))
@pytest.mark.parametrize("chain", list(CHAINS))
def test_chain_matches_cpu_fp64_graph(chain, grp, dtype):
    kinds, fn, sop = CHAINS[chain]
    rng = np.random.default_rng(zlib.crc32(f"{chain}/{grp}".encode()))
    ins = []
    for kind in kinds:
        ins.append(edge_group(rng, grp) if kind == "G" else edge_algebra(rng, grp) if kind == "A"
                   else rng.standard_normal((ins[0].shape[0], 3)))
    with torch.no_grad():
        width = _raw(fn(grp, *[torch.from_numpy(a).cuda() for a in ins])).shape[-1]
    cot = rng.standard_normal((ins[0].shape[0], width))
    compare_with_cpu_graph(lambda *t: fn(grp, *t), ins, cot, dtype, f"chain {chain} {grp} {dtype}", grp, sop,
                           scale_ins=[O.exp(grp, a) if k == "A" else a for a, k in zip(ins, kinds)])


@GPU
def test_exp_log_million_rows_fp32_forward_and_backward():
    """SE3 Exp -> Log forward + backward at 10^6 rows in fp32 (the bench row's shape): the backward kernels run
    through multi-round TMA launches from autograd.  Against the same graph in fp64 on CPU."""
    from tests.util import rand_algebra
    n = 1_000_000
    rng = np.random.default_rng(3)
    x64 = rand_algebra(rng, "SE3", n)
    cot = rng.standard_normal((n, 6))
    fn = lambda x: _lt(x, "SE3", True).Exp().Log()
    out, (gx,), (xt,) = run_graph(fn, [x64], cot, "cuda", F32)
    torch.cuda.synchronize()
    xr = _np(xt)
    cot_r = _np(torch.from_numpy(cot).float())
    with O.wide_taylor():
        X = O.exp("SE3", xr)
        y = O.log("SE3", X)
        g = O.exp_bwd("SE3", xr, O.log_bwd("SE3", y, cot_r))
    s = term_scale("SE3", "exp_fwd", [xr])
    check(_np(out), y, TOL[F32], "1e6 Exp->Log out", s)
    check(_np(gx), g, TOL[F32], "1e6 Exp->Log dx", s * (1 + np.abs(cot_r).max(1, keepdims=True)))


# ---------------------------------------------------------------------------------------------------------------------
# broadcasting
# ---------------------------------------------------------------------------------------------------------------------
def _bcast_cases(grp, rng):
    D, K = GROUPS[grp][1], GROUPS[grp][2]
    X = lambda *s: edge_group(rng, grp, n_rand=int(np.prod(s)), thetas=()).reshape(*s, D)
    big = np.concatenate([X(9), rng.standard_normal((9, 5))], 1)
    return {
        # name: (inputs, function of the torch leaves, op)
        "act_B1_1N": ([X(4, 1), rng.standard_normal((1, 5, 3))], lambda X, p: _lt(X, grp).Act(p), "act"),
        "mul_B1_1N": ([X(4, 1), X(1, 5)], lambda X, Y: _lt(X, grp) @ _lt(Y, grp), "mul"),
        "adj_D_NK": ([X(1)[0], rng.standard_normal((6, 2, K))], lambda X, a: _lt(X, grp).Adj(a), "adj"),
        "jinvp_D_NK": ([X(1)[0], rng.standard_normal((6, 2, K))], lambda X, p: _lt(X, grp).Jinvp(p), "jinvp"),
        "act4_0d": ([X(1)[0], rng.standard_normal(4)], lambda X, p: _lt(X, grp).Act(p), "act4"),
        "mul_0d": ([X(1)[0], X(1)[0]], lambda X, Y: _lt(X, grp) @ _lt(Y, grp), "mul"),
        # non-contiguous: rows of X with a stride of D + 5 elements, p as the transpose of a (3, N) tensor
        "act_strided": ([big, rng.standard_normal((3, 9))],
                        lambda B, P: _lt(B[:, :D], grp).Act(P.t()), "act"),
    }


@GPU
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("grp", list(GROUPS))
def test_broadcast_gradients_are_summed_and_match_cpu_graph(grp, dtype):
    rng = np.random.default_rng(zlib.crc32(f"bcast/{grp}".encode()))
    for name, (ins, fn, op) in _bcast_cases(grp, rng).items():
        with torch.no_grad():
            shape = _raw(fn(*[torch.from_numpy(a).cuda() for a in ins])).shape
        cot = rng.standard_normal(tuple(shape))
        if name == "act_strided":
            ts = [torch.from_numpy(a).cuda().to(dtype) for a in ins]
            assert not ts[0][:, :GROUPS[grp][1]].is_contiguous() and not ts[1].t().is_contiguous()
        grads = compare_with_cpu_graph(fn, ins, cot, dtype, f"bcast {name} {grp} {dtype}", grp, op,
                                       scale_ins=[a[:, :GROUPS[grp][1]] if name == "act_strided" and a.shape[1] > 3
                                                  else a for a in ins])
        # against the op on materialised copies: the broadcast operand's gradient is the sum over its copies
        ts = [torch.from_numpy(a).to("cuda", dtype).requires_grad_() for a in ins]
        if name != "act_strided":
            bshape = torch.broadcast_shapes(*[t.shape[:-1] for t in ts])
            mats = [t.detach().expand(bshape + t.shape[-1:]).contiguous().requires_grad_() for t in ts]
            out = _raw(fn(*mats))
            gm = torch.autograd.grad(out, mats, torch.from_numpy(cot).to("cuda", dtype))
            for t, g, m in zip(ts, grads, gm):
                lead = m.dim() - t.dim()
                s = m.sum(tuple(range(lead))) if lead else m
                dims = tuple(i for i in range(t.dim() - 1) if t.shape[i] == 1 and s.shape[i] != 1)
                s = s.sum(dims, keepdim=True) if dims else s
                tol = 1e-12 if dtype == F64 else 1e-5
                torch.testing.assert_close(g, s, rtol=tol, atol=tol * (1 + s.abs().max().item()))


# ---------------------------------------------------------------------------------------------------------------------
# torch.func and friends on CUDA
# ---------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("grp", list(GROUPS))
def test_functorch_jacobians_match_autograd_and_cpu_graph(grp, dtype):
    D, K = GROUPS[grp][1], GROUPS[grp][2]
    rng = np.random.default_rng(zlib.crc32(f"func/{grp}".encode()))
    Xn = edge_group(rng, grp, n_rand=2, thetas=(1e-3, 0.01 * (1 + 1e-3)), per=1)
    xn = edge_algebra(rng, grp, n_rand=2, thetas=(1e-3, 0.01 * (1 - 1e-3)), per=1)
    tol = dict(rtol=0, atol=1e-12) if dtype == F64 else dict(rtol=0, atol=2e-5)
    cases = {"Log": (lambda t: _lt(t, grp).Log().tensor(), Xn), "Inv": (lambda t: _lt(t, grp).Inv().tensor(), Xn),
             "Exp": (lambda t: _lt(t, grp, True).Exp().tensor(), xn)}
    for name, (f, a) in cases.items():
        t = torch.from_numpy(a).to("cuda", dtype)
        J1 = torch.func.jacrev(f)(t)
        J2 = torch.autograd.functional.jacobian(f, t, vectorize=True)
        J3 = torch.autograd.functional.jacobian(f, t)                    # plain autograd, one row at a time
        J4 = pp.func.jacrev(lambda u: f(u.tensor()))(_lt(t, grp, name == "Exp"))
        with O.wide_taylor():
            Jh = torch.func.jacrev(f)(t.double().cpu())
        for J in (J1, J2, J4):
            torch.testing.assert_close(J.double().cpu(), J3.double().cpu(), **tol)
        torch.testing.assert_close(J3.double().cpu(), Jh, **tol)
    # vmap of Act over a leading dimension, against the batched call and the CPU graph
    Xb = torch.from_numpy(edge_group(rng, grp, n_rand=6, thetas=())).to("cuda", dtype)
    p = torch.randn(6, 5, 3, dtype=dtype, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    f = lambda a, b: _lt(a, grp).Act(b)
    out = torch.vmap(f)(Xb, p)
    torch.testing.assert_close(out, f(Xb[:, None], p), rtol=0, atol=tol["atol"] * 10)
    with O.wide_taylor():
        ref = torch.vmap(f)(Xb.double().cpu(), p.double().cpu())
    torch.testing.assert_close(out.double().cpu(), ref, rtol=0, atol=tol["atol"] * 10)
    # jacrev of vmap(Act) with respect to X: the vmap rule and the backward together
    Jv = torch.func.jacrev(lambda a: torch.vmap(f)(a, p))(Xb)
    Ja = torch.autograd.functional.jacobian(lambda a: f(a[:, None], p), Xb)
    torch.testing.assert_close(Jv, Ja, rtol=0, atol=tol["atol"] * 10)


@GPU
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_modjac_on_cuda_parameter_matches_autograd_and_cpu(dtype):
    class Net(torch.nn.Module):
        def __init__(self, pose):
            super().__init__()
            self.pose = pp.Parameter(pose)

        def forward(self, x):
            return (self.pose @ x).Log().tensor()
    rng = np.random.default_rng(7)
    P, X = (torch.from_numpy(edge_group(rng, "SE3", n_rand=3, thetas=(1e-3,), per=1)) for _ in range(2))
    tol = dict(rtol=0, atol=1e-12) if dtype == F64 else dict(rtol=0, atol=2e-5)
    dev = pp.SE3(P.to("cuda", dtype)), pp.SE3(X.to("cuda", dtype))
    net = Net(dev[0])
    assert net.pose.is_cuda
    J1 = pp.optim.functional.modjac(net, input=dev[1], flatten=True, vectorize=True)
    J2 = pp.optim.functional.modjac(net, input=dev[1], flatten=True, vectorize=False)
    with O.wide_taylor():
        Jh = pp.optim.functional.modjac(Net(pp.SE3(dev[0].double().cpu())), input=pp.SE3(dev[1].double().cpu()),
                                        flatten=True, vectorize=True)
    assert J1.shape == (24, 28) and (J1[:, 6::7] == 0).all()
    torch.testing.assert_close(J1, J2, **tol)
    torch.testing.assert_close(J1.double().cpu(), Jh, **tol)


# ---------------------------------------------------------------------------------------------------------------------
# half precision: inputs are upcast to fp32 for the kernels, outputs and gradients cast back
# ---------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("grp", list(GROUPS))
def test_half_precision_keeps_dtype_and_rounds_once(grp, dtype):
    """Exp (unary) and Act (binary) against the fp64 graph of the rounded inputs and cotangent.  Outputs: within one
    rounding to `dtype` (u = 2^-11 fp16, 2^-8 bf16, relative) plus the fp32 kernels' 2e-6 term_scale bound.
    Gradients: within u (|truth| + term_scale (1 + |g|)), because the backward reads operands saved in `dtype` (Act
    saves its rounded output; gX = g @ [I, -out^, out] is a sum of such terms) and its result is rounded once more.
    Measured on an H100 SXM as a fraction of the bound: outputs 0.91 (one rounding alone may reach u), gradients 0.36."""
    u = 2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8
    rng = np.random.default_rng(zlib.crc32(f"half/{grp}".encode()))
    K = GROUPS[grp][2]
    x = edge_algebra(rng, grp, thetas=(1e-3, 0.5), per=2) * 0.5
    X = edge_group(rng, grp, thetas=(1e-3, 0.5), per=2)
    p = rng.standard_normal((X.shape[0], 3))
    for name, ins, op in (("Exp", [x], "exp"), ("Act", [X, p], "act")):
        fn = lambda *t: OPS[name][1](grp, *t)
        ts = [torch.from_numpy(a).to("cuda", dtype).requires_grad_() for a in ins]
        out = _raw(fn(*ts))
        cot = torch.randn(out.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(1)).to(dtype)
        grads = torch.autograd.grad(out, ts, cot)
        assert out.dtype == dtype and all(g.dtype == dtype for g in grads)
        _, grads_h, hs = run_graph(fn, [_np(t) for t in ts], _np(cot), "cpu", F64, wide=True)
        out_h = _raw(fn(*[h.detach() for h in hs]))
        s = term_scale(grp, f"{op}_fwd", [h.detach().numpy() for h in hs])
        for what, r, t, sc in [("out", out, out_h, s)] + [
                (f"d{i}", g, gh, s * (1 + _np(cot).__abs__().max())) for i, (g, gh) in enumerate(zip(grads, grads_h))]:
            r, t = _np(r), _np(t)
            bound = u * np.abs(t) + 2e-6 * sc if what == "out" else u * (np.abs(t) + sc)
            frac = float((np.abs(r - t) / bound).max())
            _report(f"half {grp} {name} {str(dtype)[6:]} {what}", frac)
            assert frac <= 1, f"half {grp} {name} {dtype} {what}: {np.abs(r - t).max():.3e} is {frac:.2f} of the bound"


# ---------------------------------------------------------------------------------------------------------------------
# Jinvp's group gradient (_jinvp_composite.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dev,dtype", _dev_params() + [pytest.param("cpu", F32, id="cpu-f32")])
@pytest.mark.parametrize("grp", list(GROUPS))
def test_jinvp_group_gradient(grp, dev, dtype):
    """d/dX of w . Jinvp(X, p) on rows dense around the composite's series switch (theta^2 = 1e-4) and at small
    angles, with |tau| ~ 5 for SE3 / Sim3.  SO3, RxSO3, SE3 against left-tangent differences of the exact forward;
    Sim3 against the reference-defined gradient (module docstring).  fp32 inputs are judged like fp64 ones, relative
    to (1 + |truth|) at TOL_FD[fp64]: the gradient is evaluated in fp64 from the rounded inputs.  Before it was, fp32 SE3 rows
    at theta = 0.0101 were off by 2e-2.  (cpu-f32: the CPU oracle's own fp32 Log is not a kernel under test, so
    only dX is asserted there.)"""
    K = GROUPS[grp][2]
    rng = np.random.default_rng(zlib.crc32(f"jinvp/{grp}".encode()))
    thetas = np.concatenate([0.01 * (1 + np.array([-1e-2, -1e-3, -1e-6, 1e-6, 1e-3, 1e-2])),
                             [1e-4, 3e-4, 1e-3, 3e-3, 0.02, 0.03, 0.1]])
    X = edge_group(rng, grp, thetas=thetas, per=3, n_rand=8, t_sigma=5.0)
    X = np.asarray(torch.from_numpy(X).to(dtype).double())
    p = np.asarray(torch.from_numpy(rng.standard_normal((X.shape[0], K))).to(dtype).double())
    w = rng.standard_normal((X.shape[0], K))
    w = np.asarray(torch.from_numpy(w).to(dtype).double())
    _, (gX, gp), _ = run_graph(lambda X, p: _lt(X, grp).Jinvp(p), [X, p], w, dev, dtype)
    gX = _np(gX)
    assert (gX[:, K:] == 0).all()
    truth_X = series_gradient("Jinvp", 0, [X, p], w) if grp == "Sim3" else fd_gradients(grp, "Jinvp", [X, p], w)[0]
    check(gX[:, :K], truth_X, TOL_FD[F64], f"jinvp {grp} {dev}-{dtype} dX")
    if dev == "cpu" and dtype == F32:
        return
    gp_truth = fd_gradients(grp, "Jinvp", [X, p], w)[1]
    scale = 1.0 if dtype == F64 else fp32_scale(grp, "jinvp", [X, p], w)
    check(_np(gp), gp_truth, TOL_FD[dtype], f"jinvp {grp} {dev}-{dtype} dp", scale)
