"""Gradients through pp.module.ICP on the GPU (csrc/knn.cu b200_icp_rec / b200_icp_bwd) against the reference's autograd
(tests/golden/icp_grad.npz) and its fp64 model (oracle/icp_grad_oracle.py)."""
import math

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import icp_grad_oracle as O
from tests.test_icp_grad import NAMES, golden_case

pytestmark = pytest.mark.gpu
DEV = "cuda"


def stepper(steps=15, **kw):
    return pp.utils.ReduceToBason(steps=steps, **kw)


def fixed(K):
    """exactly K iterations: tolerance and patience that cannot be met"""
    return pp.utils.ReduceToBason(steps=K, patience=10 ** 6, decreasing=-math.inf, tol=-1.0)


class HostStepper(pp.utils.ReduceToBason):
    """the same rule, run by the host loop (any stepper that is not exactly ReduceToBason)"""


def run(src, tgt, init, o, st, loss, W, probe, w, dtype):
    s = src.to(DEV, dtype).requires_grad_()
    t = tgt.to(DEV, dtype).requires_grad_()
    i = pp.SE3(init.to(DEV, dtype)).requires_grad_() if init is not None else None
    T = pp.module.ICP(stepper=st)(s, t, ord=o, init=i)
    L = (T.matrix() * W.to(DEV, dtype)).sum() if loss == 0 else (T.unsqueeze(-2).Act(probe.to(DEV, dtype)) * w.to(DEV, dtype)).sum()
    L.backward()
    return T.detach(), s.grad, t.grad, None if i is None else i.grad


def close(got, want, rtol):
    got, want = got.detach().double().cpu(), torch.as_tensor(want).double()
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= rtol, err


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("loss", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_gradients_match_reference(name, loss, dtype):
    src, tgt, init, o, K, T = golden_case(name)
    st = stepper()
    res, gs, gt, gi = run(src, tgt, init, o, st, loss, T("W"), T("probe"), T("w"), dtype)
    if dtype == torch.float32 and st.steps != K:
        pytest.skip(f"fp32 ran {st.steps} iterations, the reference {K}")
    assert st.steps == K
    rtol = 1e-8 if dtype == torch.float64 else 1e-3
    close(gs, T(f"gsrc{loss}"), rtol)
    close(gt, T(f"gtgt{loss}"), rtol)
    if init is not None:
        close(gi, T(f"ginit{loss}"), rtol)


@pytest.mark.parametrize("host_loop", [False, True])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_forward_bit_identical_with_and_without_grad(host_loop, dtype):
    src, tgt, init, o, K, T = golden_case("batched_init_o2")
    mk = (lambda: HostStepper(steps=15)) if host_loop else (lambda: stepper())
    s, t = src.to(DEV, dtype), tgt.to(DEV, dtype)
    i = pp.SE3(init.to(DEV, dtype))
    a = pp.module.ICP(stepper=mk())(s, t, init=i)
    st = mk()
    b = pp.module.ICP(stepper=st)(s.clone().requires_grad_(), t, init=i)
    assert b.requires_grad and torch.equal(a.tensor(), b.detach().tensor()) and st.steps >= 2


def test_host_loop_gradients_equal_device_loop():
    src, tgt, init, o, K, T = golden_case("bcast_tgt_init_o1")
    a = run(src, tgt, init, o, stepper(), 1, T("W"), T("probe"), T("w"), torch.float64)
    b = run(src, tgt, init, o, HostStepper(steps=15), 1, T("W"), T("probe"), T("w"), torch.float64)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_backward_is_bit_reproducible(dtype):
    g = torch.Generator().manual_seed(3)
    src = torch.rand(4, 3000, 3, generator=g, dtype=torch.float64) * 2 - 1
    tgt = src[:, :2500] @ O.quat2mat(torch.tensor([0.03, -0.02, 0.04, 1.0]) / 1.0015).T.double() + 0.05
    s = src.to(DEV, dtype).requires_grad_()
    t = tgt.to(DEV, dtype).requires_grad_()
    T = pp.module.ICP(stepper=stepper(20))(s, t)
    W = torch.randn(4, 4, 4, generator=g).to(DEV, dtype)
    L = (T.matrix() * W).sum()
    g1 = torch.autograd.grad(L, [s, t], retain_graph=True)
    g2 = torch.autograd.grad(L, [s, t])
    for x, y in zip(g1, g2):
        assert torch.isfinite(x).all() and torch.equal(x, y)


@pytest.mark.parametrize("B,N", [(3, 200), (2, 5000)])
def test_gradients_match_oracle(B, N):
    """Larger clouds than the goldens (several 1024-point CTAs per batch element) against the fp64 model."""
    g = torch.Generator().manual_seed(B * N)
    src = torch.rand(B, N, 3, generator=g, dtype=torch.float64) * 2 - 1
    R = O.quat2mat(torch.tensor([0.04, -0.02, 0.03, 1.0], dtype=torch.float64) / 1.00145)
    tgt = src @ R.T + 0.1 + 0.002 * torch.randn(B, N, 3, generator=g, dtype=torch.float64)
    init = pp.randn_SE3(B, sigma=0.01, dtype=torch.float64).tensor()
    W, probe, w = torch.randn(B, 4, 4, generator=g, dtype=torch.float64), torch.randn(B, 3, 3, generator=g, dtype=torch.float64), \
        torch.randn(B, 3, 3, generator=g, dtype=torch.float64)
    st = stepper(10)
    res, gs, gt, gi = run(src, tgt, init, 2, st, 0, W, probe, w, torch.float64)
    _, (os_, ot, oi) = O.grads(src.to(DEV), tgt.to(DEV), st.steps, init.to(DEV), 2, "project", W.to(DEV), probe.to(DEV),
                               w.to(DEV), 0)
    close(gs, os_.cpu(), 1e-8)
    close(gt, ot.cpu(), 1e-8)
    close(gi, oi.cpu(), 1e-8)


def test_target_matched_by_many_sources_gets_the_full_sum():
    g = torch.Generator().manual_seed(5)
    src = torch.rand(2, 2000, 3, generator=g, dtype=torch.float64) * 2 - 1
    tgt = torch.cat([src[:, :20] * 1.02 + 0.01, torch.full((2, 5, 3), 50.0, dtype=torch.float64)], 1)   # 20 hubs, 5 far
    W = torch.randn(2, 4, 4, generator=g, dtype=torch.float64)
    st = stepper(5)
    probe = torch.zeros(2, 1, 3, dtype=torch.float64)
    _, gs, gt, _ = run(src, tgt, None, 2, st, 0, W, probe, probe, torch.float64)
    _, (os_, ot, _) = O.grads(src.to(DEV), tgt.to(DEV), st.steps, None, 2, "project", W.to(DEV), probe.to(DEV),
                              probe.to(DEV), 0)
    close(gs, os_.cpu(), 1e-8)
    close(gt, ot.cpu(), 1e-8)
    assert (gt[:, 20:] == 0).all()


def test_planar_and_collinear_clouds():
    """Planar: finite gradients, bit-reproducible.  Collinear source: the closing Kabsch step is rank 1, so a loss on the
    returned rotation alone has zero gradient everywhere (rank <= 1: no rotation gradient; translation gets none)."""
    g = torch.Generator().manual_seed(6)
    pl = torch.rand(2, 400, 3, generator=g, dtype=torch.float64) * 2 - 1
    pl[..., 2] = 0
    R = O.quat2mat(torch.tensor([0.02, 0.01, 0.05, 1.0], dtype=torch.float64) / 1.00152)
    s = pl.to(DEV).requires_grad_()
    t = (pl @ R.T + 0.05).to(DEV).requires_grad_()
    T = pp.module.ICP(stepper=stepper(10))(s, t)
    L = (T.matrix() * torch.randn(2, 4, 4, generator=g, dtype=torch.float64).to(DEV)).sum()
    a = torch.autograd.grad(L, [s, t], retain_graph=True)
    b = torch.autograd.grad(L, [s, t])
    assert all(torch.isfinite(x).all() and torch.equal(x, y) for x, y in zip(a, b))
    line = torch.linspace(-1, 1, 300, dtype=torch.float64)[:, None] * torch.tensor([1.0, 0.5, -0.2], dtype=torch.float64)
    s = line.expand(2, 300, 3).to(DEV).requires_grad_()
    t = (line @ R.T + 0.05).expand(2, 300, 3).to(DEV).requires_grad_()
    T = pp.module.ICP(stepper=stepper(10))(s, t)
    gs, gt = torch.autograd.grad(T.tensor()[..., 3:].sum(), [s, t])
    assert (gs == 0).all() and (gt == 0).all()
    T = pp.module.ICP(stepper=stepper(10))(s, t)
    gs, gt = torch.autograd.grad(T.tensor()[..., :3].sum(), [s, t])
    assert torch.isfinite(gs).all() and torch.isfinite(gt).all() and gs.abs().max() > 0


def test_convention_mixed_graph_is_not_the_true_derivative():
    """The reference's graph feeds SE3 Act's tangent gradient into mat2SE3 as if it were Euclidean, so its gradient is
    not the derivative of the returned transform, and gradcheck of ICP as a function cannot hold: central differences
    (matches fixed under the perturbation) differ from the backward by far more than rounding."""
    g = torch.Generator().manual_seed(7)
    src = (torch.rand(1, 30, 3, generator=g, dtype=torch.float64) * 2 - 1)
    R = O.quat2mat(torch.tensor([0.05, -0.03, 0.02, 1.0], dtype=torch.float64) / 1.0019)
    tgt = src @ R.T + 0.1 + 0.005 * torch.randn(1, 30, 3, generator=g, dtype=torch.float64)
    s, t = src.to(DEV), tgt.to(DEV).requires_grad_()
    f = lambda tt: pp.module.ICP(stepper=fixed(3))(s, tt).tensor()   # noqa: E731
    ours = torch.autograd.functional.jacobian(f, t)
    num = torch.zeros_like(ours)
    h = 1e-6
    for j in range(30):
        for c in range(3):
            e = torch.zeros_like(t)
            e[0, j, c] = h
            num[..., 0, j, c] = (f(t.detach() + e) - f(t.detach() - e)) / (2 * h)
    err = float((ours - num).abs().max() / num.abs().max())
    assert err > 1e-3, err


def test_every_output_cotangent_matches_oracle():
    """The full Jacobian, one output component at a time, against the fp64 model's vector-Jacobian products."""
    g = torch.Generator().manual_seed(8)
    src = torch.rand(2, 40, 3, generator=g, dtype=torch.float64) * 2 - 1
    R = O.quat2mat(torch.tensor([0.02, -0.03, 0.01, 1.0], dtype=torch.float64) / 1.0007)
    tgt = src @ R.T + 0.05
    s, t = src.to(DEV).requires_grad_(), tgt.to(DEV).requires_grad_()
    T = pp.module.ICP(stepper=fixed(4))(s, t).tensor()
    for k in range(7):
        v = torch.zeros_like(T)
        v[:, k] = 1
        a = torch.autograd.grad(T, [s, t], v, retain_graph=True)
        Tm, _ = O.icp(s, t, 4)
        b = torch.autograd.grad(Tm, [s, t], v)
        for x, y in zip(a, b):
            close(x, y.cpu(), 1e-8)


def test_no_grad_calls_allocate_no_trace():
    g = torch.Generator().manual_seed(9)
    B, N = 2, 20000
    src = (torch.rand(B, N, 3, generator=g) * 2 - 1).to(DEV)
    tgt = src + 0.01
    icp = pp.module.ICP(stepper=fixed(8))
    icp(src, tgt)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    icp(src, tgt)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    trace_one_iteration = B * N * 4
    assert peak < trace_one_iteration, peak
    s = src.clone().requires_grad_()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    T = icp(s, tgt)
    assert torch.cuda.max_memory_allocated() - base >= 8 * trace_one_iteration
    del T
