"""GPU parity of the fused LM kernels (csrc/lm.cu) against the LM oracle and the reference's recorded
trajectories, plus convergence at the BASELINE.json sizes (configs[2] and configs[4]).

Tolerances: fp64 1e-9 relative on sums / 1e-10 on poses; fp32 1e-4 relative on sums, 5e-5 on poses.
LM converged pose error <= 1e-5 (north_star)."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch
from torch import nn

import pypose_b200 as pp
from oracle import lie_oracle as O
from oracle import lm_oracle as L
from oracle import scan_oracle as S
from tests.util import rand_group

pytestmark = pytest.mark.gpu
ops = torch.ops.b200pose
DT = [(torch.float64, 1e-9, 1e-10), (torch.float32, 2e-4, 5e-5)]


def cu(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


@pytest.mark.parametrize("dt,rtol,ptol", DT, ids=["f64", "f32"])
def test_poseinv_trial_vs_oracle(dt, rtol, ptol):
    rng = np.random.default_rng(0)
    n = 5003
    P = rand_group(rng, "SE3", n, tmax=2.0)
    X = rand_group(rng, "SE3", n, tmax=2.0)
    Pd, Xd = cu(P, dt), cu(X, dt)
    Pt, sums = ops.lm_poseinv_trial(Pd, Xd, 1.0001, 1e-6, 1e32, 0, 1.0)
    Pt_o, sums_o = L.poseinv_trial(Pd.double().cpu().numpy(), Xd.double().cpu().numpy(), 1.0001, 1e-6, 1e32)
    assert np.abs(Pt.double().cpu().numpy() - Pt_o).max() <= ptol * 20
    s = sums.cpu().numpy()
    np.testing.assert_allclose(s[0], sums_o[0], rtol=rtol)
    np.testing.assert_allclose(s[2], sums_o[2], rtol=rtol * 10)
    assert s[1] <= max(10 * sums_o[1], 1e-6 * s[0]) and s[3] == 0
    loss = ops.lm_poseinv_loss(Pd, Xd, 0, 1.0).cpu().numpy()
    np.testing.assert_allclose(loss[0], sums_o[0], rtol=rtol)


def _reproj_problem(rng, C, M, noise=0.05, pix_noise=0.0):
    gt = rand_group(rng, "SE3", C, tmax=0.5, t_sigma=0.5)
    cidx = rng.integers(0, C, M)
    cidx[:C] = np.arange(C)
    pc = rng.uniform([-2, -2, 2], [2, 2, 6], (M, 3))
    pts = O.act("SE3", O.inv("SE3", gt)[cidx], pc)
    pix = -pc[:, :2] / pc[:, 2:] + pix_noise * rng.standard_normal((M, 2))
    init = O.mul("SE3", O.exp("SE3", noise * rng.standard_normal((C, 6))), gt)
    return gt, init, pts, pix, cidx


@pytest.mark.parametrize("dt,rtol,ptol", DT, ids=["f64", "f32"])
def test_reproj_accum_solve_loss_vs_oracle(dt, rtol, ptol):
    rng = np.random.default_rng(1)
    C, M = 301, 30011
    gt, init, pts, pix, cidx = _reproj_problem(rng, C, M)
    order = np.argsort(cidx, kind="stable")
    seg = np.concatenate([[0], np.cumsum(np.bincount(cidx, minlength=C))]).astype(np.int32)
    pd, td, xd = cu(init, dt), cu(pts[order], dt), cu(pix[order], dt)
    segd, cd = torch.from_numpy(seg).cuda(), torch.from_numpy(cidx[order].astype(np.int32)).cuda()
    H, g, s = ops.lm_reproj_accum(pd, td, xd, segd, 0, 1.0)
    H_o, g_o, s_o = L.reproj_accum(pd.double().cpu().numpy(), td.double().cpu().numpy(), xd.double().cpu().numpy(), seg)
    scaleH = np.abs(H_o).max()
    assert np.abs(H.double().cpu().numpy() - H_o).max() <= rtol * scaleH
    assert np.abs(g.double().cpu().numpy() - g_o).max() <= rtol * np.abs(g_o).max()
    np.testing.assert_allclose(s.cpu().numpy()[0], s_o[0], rtol=rtol)
    Pt, D, s2 = ops.lm_solve6_retract(H, g, pd, 1.0001, 1e-6, 1e32)
    Pt_o, D_o, s2_o = L.solve6_retract(H.double().cpu().numpy(), g.double().cpu().numpy(), pd.double().cpu().numpy(),
                                       1.0001, 1e-6, 1e32)
    assert np.abs(D.double().cpu().numpy() - D_o).max() <= ptol * 100
    assert np.abs(Pt.double().cpu().numpy() - Pt_o).max() <= ptol * 100
    np.testing.assert_allclose(s2.cpu().numpy()[0], s2_o[0], rtol=rtol * 50)
    lo = ops.lm_reproj_loss(Pt, td, xd, segd, 0, 1.0).cpu().numpy()[0]
    np.testing.assert_allclose(lo, L.reproj_loss(Pt.double().cpu().numpy(), td.double().cpu().numpy(),
                                                 xd.double().cpu().numpy(), cidx[order])[0], rtol=rtol * 10, atol=1e-12)
    r = ops.lm_reproj_residual(pd, td, xd, cd)
    r_o = L.reproj_residual(pd.double().cpu().numpy(), td.double().cpu().numpy(), xd.double().cpu().numpy(), cidx[order])
    assert np.abs(r.double().cpu().numpy() - r_o).max() <= ptol


class InvNet(nn.Module):
    def __init__(self, pose):
        super().__init__()
        self.pose = pp.Parameter(pose)

    def forward(self, input):
        return (self.pose @ input).Log().tensor()


@pytest.mark.parametrize("strategy", ["constant", "trustregion", "adaptive"])
def test_lm_poseinv_reference_trajectory_on_gpu(golden_lm, strategy):
    g = golden_lm
    st = {"constant": lambda: pp.optim.strategy.Constant(damping=1e-4), "trustregion": lambda: pp.optim.strategy.TrustRegion(),
          "adaptive": lambda: pp.optim.strategy.Adaptive(damping=1e-2)}[strategy]()
    net = InvNet(pp.SE3(torch.from_numpy(g["poseinv/P0"].copy()).cuda()))
    X = pp.SE3(torch.from_numpy(g["poseinv/X"].copy()).cuda())
    opt = pp.optim.LM(net, strategy=st)
    for k in range(4):
        loss = opt.step(X)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g[f"poseinv/{strategy}/loss"][k], rtol=1e-5, atol=1e-20)
        np.testing.assert_allclose(net.pose.detach().cpu().numpy(), g[f"poseinv/{strategy}/poses"][k], atol=1e-9)
        assert opt.reject_count == g[f"poseinv/{strategy}/reject"][k]


@pytest.mark.parametrize("case,strategy,steps", [("reproj", "constant", 4), ("reproj", "trustregion", 4),
                                                 ("reproj_hard", "trustregion", 6)])
@pytest.mark.parametrize("route", ["structured", "generic"])
def test_lm_reproj_reference_trajectory_on_gpu(golden_lm, case, strategy, steps, route):
    g = golden_lm
    st = {"constant": lambda: pp.optim.strategy.Constant(damping=1e-4), "trustregion": lambda: pp.optim.strategy.TrustRegion()}[strategy]()
    net = pp.module.PoseReproj(pp.SE3(torch.from_numpy(g[f"{case}/poses0"].copy()).cuda()))
    inp = tuple(torch.from_numpy(g[f"{case}/{k}"]).cuda() for k in ("pts", "pix", "cidx"))
    opt = pp.optim.LM(net, strategy=st, solver=None if route == "structured" else pp.optim.solver.Cholesky(upper=True))
    for k in range(steps):
        loss = opt.step(inp)
        np.testing.assert_allclose(float(loss), g[f"{case}/{strategy}/loss"][k], rtol=1e-6)
        np.testing.assert_allclose(net.poses.detach().cpu().numpy(), g[f"{case}/{strategy}/poses"][k], atol=1e-8)
        assert opt.reject_count == g[f"{case}/{strategy}/reject"][k]


@pytest.mark.parametrize("dt,tol", [(torch.float64, 1e-11), (torch.float32, 2e-5)], ids=["f64", "f32"])
@pytest.mark.parametrize("kernel", [None, "huber"])
def test_reproj_staged_route_matches_register_route(dt, tol, kernel):
    """csrc/lmstep.cu reproj_trial_staged_kernel (rows through a TMA-fed shared-memory ring, one warp per camera) against the
    register-fed reproj_trial_kernel on ragged per-camera row lists: empty cameras, 1 row, lists that end exactly on a
    tile, lists shorter / longer than the ring, a total that is not a multiple of 4 (the last tile is copied by the lanes),
    accepted and rejected trials (the retry runs from the stored blocks)."""
    import ctypes
    from pypose_b200 import _C
    rng = np.random.default_rng(11)
    counts = np.array([0, 1, 3, 127, 128, 129, 511, 512, 513, 640, 2000, 0, 5, 1537, 64, 4099, 2, 0, 777, 1023], np.int64)
    C, M = counts.size, int(counts.sum())
    assert M % 4 != 0
    cidx = rng.permutation(np.repeat(np.arange(C), counts))
    gt = rand_group(rng, "SE3", C, tmax=0.5, t_sigma=0.5)
    pc = rng.uniform([-2, -2, 2], [2, 2, 6], (M, 3))
    pts = O.act("SE3", O.inv("SE3", gt)[cidx], pc)
    pix = -pc[:, :2] / pc[:, 2:] + 0.01 * rng.standard_normal((M, 2))
    if kernel:
        pix[rng.random(M) < 0.05] += 0.5
    init = O.mul("SE3", O.exp("SE3", 0.1 * rng.standard_normal((C, 6))), gt)
    inp = (cu(pts, dt), cu(pix, dt), torch.from_numpy(cidx).cuda())
    mode = _C.lib().b200_lm_reproj_staged_mode
    mode.restype, mode.argtypes = ctypes.c_int, [ctypes.c_int]
    prev = mode(-1)
    out = {}
    try:
        for m in (0, 2):
            mode(m)
            net = pp.module.PoseReproj(pp.SE3(cu(init, dt)))
            opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(radius=1e4),
                              kernel=pp.optim.kernel.Huber(delta=0.1) if kernel else None)
            losses, rejects = [], []
            for _ in range(6):
                losses.append(float(opt.step(inp)))
                rejects.append(opt.reject_count)
            out[m] = (np.array(losses), rejects, net.poses.detach().double().cpu().numpy())
    finally:
        mode(prev)
    np.testing.assert_allclose(out[2][0], out[0][0], rtol=tol * 10)
    assert out[2][1] == out[0][1]
    assert np.abs(out[2][2] - out[0][2]).max() <= tol * 10
    assert out[0][0][-1] < out[0][0][0]


def test_config3_invnet_1e5_fp32_converges():
    """BASELINE.json configs[2]: README InvNet, 1e5 SE3 poses, fp32, Constant(1e-4), Cholesky, 10 iterations.
    (rotations of the inputs are kept away from the Log branch cut, SURVEY.md §8d cfg 3.)"""
    torch.manual_seed(0)
    n = 100_000
    X = pp.randn_SE3(n, sigma=0.9, device="cuda")
    net = InvNet(pp.randn_SE3(n, sigma=0.9, device="cuda"))
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.Constant(damping=1e-4))
    for _ in range(10):
        loss = opt.step(X)
    assert opt._problem is not None
    err = (net.pose @ X).Log().tensor().abs().max().item()
    assert err <= 1e-5, err


def test_config5_reproj_1e4_poses_1e6_residuals_converges():
    """BASELINE.json configs[4] (single-pose form): 1e4 poses, 1e6 reprojection residuals, fp32."""
    rng = np.random.default_rng(3)
    C, M = 10_000, 1_000_000
    gt, init, pts, pix, cidx = _reproj_problem(rng, C, M, noise=0.05)
    net = pp.module.PoseReproj(pp.SE3(cu(init, torch.float32)))
    inp = (cu(pts, torch.float32), cu(pix, torch.float32), torch.from_numpy(cidx).cuda())
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion())
    l0 = None
    for _ in range(10):
        loss = float(opt.step(inp))
        l0 = loss if l0 is None else l0
    assert loss < 1e-3 * l0 or loss < 1e-4
    d = (pp.SE3(cu(gt, torch.float32)).Inv() @ net.poses).Log().tensor().abs().max().item()
    print(f"config 5 (single-pose form) fp32: converged pose error max |Log(gt^-1 P)| = {d:.3e}, loss {loss:.3e}")
    assert d <= 1e-5, d           # north_star's bound, in fp32 at the full size


def test_config5_small_fp64_pose_error():
    rng = np.random.default_rng(4)
    C, M = 500, 50_000
    gt, init, pts, pix, cidx = _reproj_problem(rng, C, M, noise=0.05)
    net = pp.module.PoseReproj(pp.SE3(cu(init, torch.float64)))
    inp = (cu(pts, torch.float64), cu(pix, torch.float64), torch.from_numpy(cidx).cuda())
    opt = pp.optim.LM(net)
    for _ in range(8):
        opt.step(inp)
    d = (pp.SE3(cu(gt, torch.float64)).Inv() @ net.poses).Log().tensor().abs().max().item()
    assert d <= 1e-5, d


@pytest.mark.parametrize("kname,kern", [("huber", lambda: pp.optim.kernel.Huber(delta=0.05)),
                                        ("cauchy", lambda: pp.optim.kernel.Cauchy(delta=0.1)),
                                        ("pseudohuber", lambda: pp.optim.kernel.PseudoHuber(delta=0.05)),
                                        ("softlone", lambda: pp.optim.kernel.SoftLOne(delta=0.1)),
                                        ("arctan", lambda: pp.optim.kernel.Arctan(delta=0.3))])
def test_lm_robust_kernels_reference_trajectory_on_gpu(golden_lm, kname, kern):
    g = golden_lm
    net = pp.module.PoseReproj(pp.SE3(torch.from_numpy(g["robust_reproj/poses0"].copy()).cuda()))
    inp = tuple(torch.from_numpy(g[f"robust_reproj/{k}"]).cuda() for k in ("pts", "pix", "cidx"))
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), kernel=kern())
    for k in range(5):
        loss = opt.step(inp)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g[f"robust_reproj/{kname}/loss"][k], rtol=1e-6)
        np.testing.assert_allclose(net.poses.detach().cpu().numpy(), g[f"robust_reproj/{kname}/poses"][k], atol=1e-8)
        assert opt.reject_count == g[f"robust_reproj/{kname}/reject"][k]


@pytest.mark.parametrize("kind,delta", [(1, 0.05), (2, 0.05), (3, 0.1), (4, 0.1), (5, 0.3), (6, 0.5)])
def test_robust_accum_and_poseinv_vs_oracle(kind, delta):
    rng = np.random.default_rng(kind)
    C, M = 101, 9001
    gt, init, pts, pix, cidx = _reproj_problem(rng, C, M, pix_noise=0.05)
    order = np.argsort(cidx, kind="stable")
    seg = np.concatenate([[0], np.cumsum(np.bincount(cidx, minlength=C))]).astype(np.int32)
    dt = torch.float64
    pd, td, xd = cu(init, dt), cu(pts[order], dt), cu(pix[order], dt)
    H, g, s = ops.lm_reproj_accum(pd, td, xd, torch.from_numpy(seg).cuda(), kind, delta)
    H_o, g_o, s_o = L.reproj_accum(init, pts[order], pix[order], seg, kind, delta)
    assert np.abs(H.cpu().numpy() - H_o).max() <= 1e-9 * np.abs(H_o).max()
    assert np.abs(g.cpu().numpy() - g_o).max() <= 1e-9 * np.abs(g_o).max()
    np.testing.assert_allclose(s.cpu().numpy()[0], s_o[0], rtol=1e-10)
    P, X = rand_group(rng, "SE3", 2001, tmax=2.0), rand_group(rng, "SE3", 2001, tmax=2.0)
    Pt, sums = ops.lm_poseinv_trial(cu(P, dt), cu(X, dt), 1.0001, 1e-6, 1e32, kind, delta)
    Pt_o, sums_o = L.poseinv_trial(P, X, 1.0001, 1e-6, 1e32, kind, delta)
    assert np.abs(Pt.cpu().numpy() - Pt_o).max() <= 1e-9
    np.testing.assert_allclose(sums.cpu().numpy()[:3], sums_o[:3], rtol=1e-8)


def _pgo_problem(rng, N, extra, noise=0.1, meas_noise=0.0, span=None):
    """A long noisy trajectory with odometry edges plus `extra` loop closures between random nodes, or with `span`
    between nodes at most `span` apart (a banded H)."""
    step = O.exp("SE3", np.tile(np.array([[1.0, 0.1, 0.0, 0.0, 0.0, 0.2]]), (N, 1)) + 0.05 * rng.standard_normal((N, 6)))
    gt = step.copy()
    d = 1
    while d < N:                          # gt[i] = step[0] ... step[i] by log2(N) vectorised doubling steps
        gt[d:] = O.mul("SE3", gt[:-d], gt[d:])
        d *= 2
    if span:
        ci = rng.integers(0, N - span, extra)
        cj = ci + rng.integers(2, span + 1, extra)
    else:
        ci, cj = rng.integers(0, N, extra), rng.integers(0, N, extra)
    ei, ej = np.concatenate([np.arange(N - 1), ci]), np.concatenate([np.arange(1, N), cj])
    keep = ei != ej
    ei, ej = ei[keep], ej[keep]
    Z = O.mul("SE3", O.inv("SE3", gt[ei]), gt[ej])
    if meas_noise:
        Z = O.mul("SE3", O.exp("SE3", meas_noise * rng.standard_normal((len(ei), 6))), Z)
    init = O.mul("SE3", O.exp("SE3", noise * rng.standard_normal((N, 6))), gt)
    return gt, init, np.stack([ei, ej], 1), Z


def test_pgo_kernels_vs_oracle():
    rng = np.random.default_rng(8)
    gt, init, edges, Z = _pgo_problem(rng, 400, 300, meas_noise=0.02)
    dt = torch.float64
    nd, Zd = cu(init, dt), cu(Z, dt)
    ei, ej = (torch.from_numpy(edges[:, k].astype(np.int32)).cuda() for k in (0, 1))
    for kind, delta in ((0, 1.0), (1, 0.1)):
        M, u, c = ops.lm_pgo_linearize(nd, Zd, ei, ej, kind, delta)
        M_o, u_o, c_o = L.pgo_linearize(init, Z, edges[:, 0], edges[:, 1], kind, delta)
        assert np.abs(M.cpu().numpy() - M_o).max() <= 1e-9 * np.abs(M_o).max()
        assert np.abs(u.cpu().numpy() - u_o).max() <= 1e-9 * max(1.0, np.abs(u_o).max())
        np.testing.assert_allclose(c.cpu().numpy()[0], c_o[0], rtol=1e-10)
    Hd, g = ops.lm_pgo_scatter(M, u, ei, ej, 400)
    Hd_o, g_o = L.pgo_scatter(M_o, u_o, edges[:, 0], edges[:, 1], 400)
    assert np.abs(Hd.cpu().numpy() - Hd_o).max() <= 1e-9 * np.abs(Hd_o).max()
    assert np.abs(g.cpu().numpy() - g_o).max() <= 1e-9 * np.abs(g_o).max()
    x = rng.standard_normal((400, 6))
    y = ops.lm_pgo_spmv(M, ei, ej, cu(x, dt), torch.zeros(400, 6, dtype=dt, device="cuda"))
    y_o = L.pgo_spmv(M_o, edges[:, 0], edges[:, 1], x, np.zeros((400, 6)))
    assert np.abs(y.cpu().numpy() - y_o).max() <= 1e-9 * np.abs(y_o).max()
    lo = ops.lm_pgo_loss(nd, Zd, ei, ej, 0, 1.0).cpu().numpy()[0]
    np.testing.assert_allclose(lo, L.pgo_loss(init, Z, edges[:, 0], edges[:, 1])[0], rtol=1e-10)


@pytest.mark.parametrize("strategy", ["constant", "trustregion"])
def test_lm_pgo_reference_trajectory_on_gpu(golden_lm, strategy):
    g = golden_lm
    st = {"constant": lambda: pp.optim.strategy.Constant(damping=1e-4), "trustregion": lambda: pp.optim.strategy.TrustRegion()}[strategy]()
    net = pp.module.PoseGraph(pp.SE3(torch.from_numpy(g["pgo/nodes0"].copy()).cuda()))
    inp = (torch.from_numpy(g["pgo/edges"]).cuda(), pp.SE3(torch.from_numpy(g["pgo/Z"].copy()).cuda()))
    opt = pp.optim.LM(net, strategy=st, solver=pp.optim.solver.PCG(tol=1e-12), sparse=True)
    for k in range(5):
        loss = opt.step(inp)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g[f"pgo/{strategy}/loss"][k], rtol=1e-6)
        np.testing.assert_allclose(net.nodes.detach().cpu().numpy(), g[f"pgo/{strategy}/poses"][k], atol=1e-7)
        assert opt.reject_count == g[f"pgo/{strategy}/reject"][k]


def test_pgo_large_graph_fp32_converges():
    """2e4 nodes / 6e4 edges, fp32, PCG(tol=1e-4): the loss drops by > 1e3x and every edge error ends < 1e-2
    (the reference's dense route would need a 1.2e5 x 1.4e5 Jacobian; its sparse route needs `bae`)."""
    rng = np.random.default_rng(9)
    N = 20_000
    gt, init, edges, Z = _pgo_problem(rng, N, 2 * N, noise=0.05)
    net = pp.module.PoseGraph(pp.SE3(cu(init, torch.float32)))
    inp = (torch.from_numpy(edges).cuda(), pp.SE3(cu(Z, torch.float32)))
    opt = pp.optim.LM(net, solver=pp.optim.solver.PCG(tol=1e-4, maxiter=200), sparse=True)
    losses = [float(opt.step(inp)) for _ in range(8)]
    assert losses[-1] < 1e-3 * losses[0] or losses[-1] < 1e-4, losses
    assert net(*inp).abs().max().item() < 1e-2


def _ba_problem(rng, C, P, per_point, noise_T=0.02, noise_p=0.05, pix_noise=0.0, consecutive=False):
    """Point j is seen by `per_point` cameras: j, j+1, ... (mod C) if `consecutive` (a banded Schur complement), else
    spread out."""
    gt = rand_group(rng, "SE3", C, tmax=0.3, t_sigma=0.3)
    ptsw = rng.uniform([-2, -2, 3], [2, 2, 6], (P, 3))
    if consecutive:
        cidx = (np.repeat(np.arange(P), per_point) + np.tile(np.arange(per_point), P)) % C
    else:
        cidx = (np.repeat(np.arange(P), per_point) * 7 + np.tile(np.arange(per_point), P) * 3) % C
    pidx = np.repeat(np.arange(P), per_point)
    y = O.act("SE3", gt[cidx], ptsw[pidx])
    pix = -y[:, :2] / y[:, 2:] + pix_noise * rng.standard_normal((len(cidx), 2))
    T0 = O.mul("SE3", O.exp("SE3", noise_T * rng.standard_normal((C, 6))), gt)
    p0 = ptsw + noise_p * rng.standard_normal((P, 3))
    return gt, ptsw, T0, p0, pix, cidx, pidx


def test_ba_kernels_vs_oracle():
    rng = np.random.default_rng(15)
    gt, ptsw, T0, p0, pix, cidx, pidx = _ba_problem(rng, 40, 900, 4, pix_noise=0.01)
    dt = torch.float64
    ci, pi_ = torch.from_numpy(cidx.astype(np.int32)).cuda(), torch.from_numpy(pidx.astype(np.int32)).cuda()
    for kind, delta in ((0, 1.0), (1, 0.02)):
        outs = ops.lm_ba_linearize(cu(T0, dt), cu(p0, dt), cu(pix, dt), ci, pi_, kind, delta)
        outs_o = L.ba_linearize(T0, p0, pix, cidx, pidx, kind, delta)
        for a, b, nm in zip(outs, outs_o, ("Jc", "Jp", "rs", "Hcc", "Hpp", "gc", "gp", "loss")):
            assert np.abs(a.cpu().numpy() - b).max() <= 1e-9 * max(1.0, np.abs(b).max()), nm
    Jc, Jp = outs[0], outs[1]
    x, v = rng.standard_normal((40, 6)), rng.standard_normal((900, 3))
    t = ops.lm_ba_wtx(Jc, Jp, ci, pi_, cu(x, dt), 900).cpu().numpy()
    y = ops.lm_ba_wv(Jc, Jp, ci, pi_, cu(v, dt), 40).cpu().numpy()
    assert np.abs(t - L.ba_wtx(outs_o[0], outs_o[1], cidx, pidx, x, 900)).max() <= 1e-9 * np.abs(t).max()
    assert np.abs(y - L.ba_wv(outs_o[0], outs_o[1], cidx, pidx, v, 40)).max() <= 1e-9 * np.abs(y).max()
    lo = ops.lm_ba_loss(cu(T0, dt), cu(p0, dt), cu(pix, dt), ci, pi_, 0, 1.0).cpu().numpy()[0]
    np.testing.assert_allclose(lo, L.ba_loss(T0, p0, pix, cidx, pidx)[0], rtol=1e-10)


@pytest.mark.parametrize("strategy", ["constant", "trustregion"])
def test_lm_bundle_adjustment_reference_trajectory_on_gpu(golden_lm, strategy):
    g = golden_lm
    st = {"constant": lambda: pp.optim.strategy.Constant(damping=1e-4), "trustregion": lambda: pp.optim.strategy.TrustRegion()}[strategy]()
    net = pp.module.BundleAdjustment(pp.SE3(torch.from_numpy(g["ba/poses0"].copy()).cuda()),
                                     torch.from_numpy(g["ba/points0"].copy()).cuda())
    inp = tuple(torch.from_numpy(g[f"ba/{k}"]).cuda() for k in ("pix", "cidx", "pidx"))
    opt = pp.optim.LM(net, strategy=st, solver=pp.optim.solver.PCG(tol=1e-12), sparse=True)
    for k in range(5):
        loss = opt.step(inp)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g[f"ba/{strategy}/loss"][k], rtol=1e-5)
        np.testing.assert_allclose(net.poses.detach().cpu().numpy(), g[f"ba/{strategy}/poses"][k], atol=1e-6)
        np.testing.assert_allclose(net.points_3d.detach().cpu().numpy(), g[f"ba/{strategy}/points"][k], atol=1e-6)
        assert opt.reject_count == g[f"ba/{strategy}/reject"][k]


def test_ba_large_fp32_converges():
    """300 cameras, 60 k points, 4.8e5 observations, fp32, Schur PCG(tol 1e-4): loss drops > 1e3x."""
    rng = np.random.default_rng(16)
    gt, ptsw, T0, p0, pix, cidx, pidx = _ba_problem(rng, 300, 60_000, 8)
    net = pp.module.BundleAdjustment(pp.SE3(cu(T0, torch.float32)), cu(p0, torch.float32))
    inp = (cu(pix, torch.float32), torch.from_numpy(cidx).cuda(), torch.from_numpy(pidx).cuda())
    opt = pp.optim.LM(net, solver=pp.optim.solver.PCG(tol=1e-4, maxiter=100), sparse=True)
    losses = [float(opt.step(inp)) for _ in range(8)]
    assert losses[-1] < 1e-3 * losses[0], losses


def _dense_sym(packed, n, k):
    """(n, k(k+1)/2) packed upper triangles -> (n,k,k)."""
    iu = np.triu_indices(k)
    A = np.zeros((n, k, k))
    A[:, iu[0], iu[1]] = packed
    A[:, iu[1], iu[0]] = packed
    return A


def test_block_damp_inverse_kernels():
    """b200_lm_blk6_damp_inv / pt3_damp_inv / pt3_apply against numpy (clamp + damping of optimizer.py:657/666)."""
    import ctypes
    from pypose_b200.optim import _fused as F
    rng = np.random.default_rng(21)
    n = 1037
    for dt, tol in ((torch.float64, 1e-9), (torch.float32, 2e-3)):
        B = rng.standard_normal((n, 6, 8))
        A = B @ B.transpose(0, 2, 1)
        A[::7, 2, :] = 0.0                                    # an unobserved direction: diagonal below the clamp,
        A[::7, :, 2] = 0.0                                    # block stays positive semi-definite
        iu = np.triu_indices(6)
        H = cu(A[:, iu[0], iu[1]], dt)
        Hd, ex, Mi = (torch.empty(n, w, dtype=dt, device="cuda") for w in (21, 6, 21))
        F._launch("b200_lm_blk6_damp_inv", H, [F._p(H), 1.5, 1e-6, 1e32, F._p(Hd), F._p(ex), F._p(Mi)], n)
        Ad = _dense_sym(H.double().cpu().numpy(), n, 6)
        d = np.einsum('nii->ni', Ad).copy()
        dd = np.clip(d, 1e-6, 1e32) * 1.5
        Ad[:, np.arange(6), np.arange(6)] = dd
        np.testing.assert_allclose(ex.double().cpu().numpy(), dd - d, rtol=1e-6, atol=1e-12)
        np.testing.assert_allclose(_dense_sym(Hd.double().cpu().numpy(), n, 6), Ad, rtol=1e-6, atol=1e-12)
        I = _dense_sym(Mi.double().cpu().numpy(), n, 6) @ Ad
        assert np.isfinite(I).all()
        well = np.ones(n, bool) if dt == torch.float64 else (np.arange(n) % 7 != 0)     # cond ~1e7 blocks: fp64 only
        assert np.abs(I[well] - np.eye(6)).max() <= tol * 10
        B3 = rng.standard_normal((n, 3, 5))
        A3 = B3 @ B3.transpose(0, 2, 1)
        iu3 = np.triu_indices(3)
        H3 = cu(A3[:, iu3[0], iu3[1]], dt)
        Hi3 = torch.empty(n, 6, dtype=dt, device="cuda")
        F._launch("b200_lm_pt3_damp_inv", H3, [F._p(H3), 1.25, 1e-6, 1e32, F._p(Hi3)], n)
        A3d = _dense_sym(H3.double().cpu().numpy(), n, 3)
        A3d[:, np.arange(3), np.arange(3)] *= 1.25
        I3 = _dense_sym(Hi3.double().cpu().numpy(), n, 3) @ A3d
        assert np.abs(I3 - np.eye(3)).max() <= tol * 10
        t = rng.standard_normal((n, 3))
        out = torch.empty(n, 3, dtype=dt, device="cuda")
        F._launch("b200_lm_pt3_apply", H3, [F._p(Hi3), F._p(cu(t, dt)), -2.0, F._p(out)], n)
        ref = -2.0 * np.einsum('nij,nj->ni', _dense_sym(Hi3.double().cpu().numpy(), n, 3), cu(t, dt).double().cpu().numpy())
        np.testing.assert_allclose(out.double().cpu().numpy(), ref, rtol=1e-5 if dt == torch.float32 else 1e-12, atol=1e-6 if dt == torch.float32 else 1e-12)


# ------------------------------------------------------------------ device PCG (csrc/pcg.cu, pcg2.cu) against fp64 sparse solves
# The solver picks its kernels from the system size n (poses or cameras).  lm_grid caps a grid at 8 CTAs per SM (1056 on
# the 132-SM H100 SXM):
#   n <= 2048 / 3072 / 4096    cg_vec_small_kernel<256 / 512 / 1024>, one CTA per iteration (scatter pose graph, BA)
#   n > 4096                   grid path cg_dot -> cg_update -> cg_dir (scatter pose graph, BA)
#   any n                      pcg2 operator + cg_update (node-ordered pose graph, the single-GPU default)
#   n > 384 * 128 = 49152      cg_update has > 384 CTAs: reduce_sums folds the partials in its kFold loop
#   n > 1056 * 128 = 135168    cg_update's grid-stride loop
PGO_N = [90, 2500, 3500, 4500, 60_000, 140_000]
# dtype, damping scale, tolerance.  fp64: barely damped, solved far below what fp32 reaches.  fp32: a well-conditioned
# version of the same system (the damping bounds the block-Jacobi preconditioned condition number by ~ 1 / (scale - 1))
# at a tolerance fp32 reaches.
PCG_DT = {"f64": (torch.float64, 1.0 + 1e-4, 1e-13), "f32": (torch.float32, 1.05, 1e-4)}
UNIT_ROUNDOFF = {torch.float64: 2.0 ** -53, torch.float32: 2.0 ** -24}


def _pgo_sparse_H(M, edges, N):
    """fp64 H = sum_e (e_i - e_j) M_e (e_i - e_j)^T (6x6 blocks) from the packed per-edge blocks M (E, 21)."""
    B = _dense_sym(M, M.shape[0], 6).reshape(-1, 36)
    a, b = np.divmod(np.arange(36), 6)
    i, j = 6 * edges[:, :1].astype(np.int64), 6 * edges[:, 1:].astype(np.int64)
    rows = np.concatenate([(p + a).ravel() for p in (i, j, i, j)])
    cols = np.concatenate([(q + b).ravel() for q in (i, j, j, i)])
    vals = np.concatenate([B.ravel(), B.ravel(), -B.ravel(), -B.ravel()])
    return sp.csr_matrix((vals, (rows, cols)), shape=(6 * N, 6 * N))


def _ba_sparse_J(Jc, Jp, cidx, pidx, C, P):
    """fp64 Jacobian (2m, 6C + 3P) of the reprojection rows from the stored rows Jc (m, 12) and Jp (m, 6)."""
    m = len(cidx)
    row = 2 * np.arange(m)[:, None, None] + np.arange(2)[None, :, None]
    rows, cols, vals = [], [], []
    for Jb, w, off, idx in ((Jc, 6, 0, cidx), (Jp, 3, 6 * C, pidx)):
        rows.append(np.broadcast_to(row, (m, 2, w)).ravel())
        cols.append(np.broadcast_to(off + w * idx.astype(np.int64)[:, None, None] + np.arange(w), (m, 2, w)).ravel())
        vals.append(Jb.reshape(m, 2, w).ravel())
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(2 * m, 6 * C + 3 * P))


def _damped(H, scale, dmin, dmax):
    """H + diag(clamp(d, dmin, dmax) scale - d), d = diag(H): the system every LM step solves (optimizer.py:657/666)."""
    d = H.diagonal()
    return (H + sp.diags(np.clip(d, dmin, dmax) * scale - d)).tocsr()


def _ref_solve(A, b, direct):
    """fp64 solution of A x = b: sparse LU where its fill stays small (banded systems of a few 1e4 unknowns), else
    Jacobi-preconditioned CG to 1e-12 (used on well-conditioned systems only)."""
    if direct:
        return spla.spsolve(A.tocsc(), b)
    x, info = spla.cg(A, b, rtol=1e-12, maxiter=20_000, M=sp.diags(1.0 / A.diagonal()))
    assert info == 0
    return x


def _ba_ref_solve(A, b, C):
    """fp64 solution of the full bundle-adjustment system A x = b (6C camera unknowns, then 3x3 point blocks): the points
    are eliminated exactly, the camera system is solved by sparse LU, then the points are substituted back."""
    n = 6 * C
    P = (A.shape[0] - n) // 3
    App = A[n:, n:].tocoo()
    B = np.zeros((P, 3, 3))
    B[App.row // 3, App.row % 3, App.col % 3] = App.data
    Pinv = sp.bsr_matrix((np.linalg.inv(B), np.arange(P), np.arange(P + 1)), shape=(3 * P, 3 * P)).tocsr()
    Acp = A[:n, n:]
    xc = spla.spsolve((A[:n, :n] - Acp @ Pinv @ Acp.T).tocsc(), b[:n] - Acp @ (Pinv @ b[n:]))
    return np.concatenate([xc, Pinv @ (b[n:] - Acp.T @ xc)])


def _check_pcg(tag, H, A, g, x, xref, scale, tol, dt, errtol):
    """x: a device PCG solution of A x = -g in `dt` (A: H damped).  Checked against bounds derived before the solve was run:
        |A x + g| / |g| <= tol + 100 u kappa,   kappa = |A|_G |x*| / |g|
    tol is the stop test on the recursive residual; 100 u kappa covers the rounding of the operator products (~30 terms
    per row of A summed in `dt`, unit roundoff u) and the drift of the recursive residual away from the true one over
    the iterations, both of order u |A| |x|.  |A|_G: the Gershgorin bound on |A|_2; x*: the fp64 reference (x itself
    where none is computed).
        |x - x*| / |x*| <= (residual bound) |g| / (lambda_min |x*|),   lambda_min >= min_i (scale - 1) d_i
    because H is positive semi-definite and the damping adds at least (scale - 1) d_i to every diagonal entry d_i
    (unknowns that no residual touches, d_i = 0, are a separate diagonal block with a zero right-hand side).
    fp64 solutions also meet the fixed `errtol`.
    Measured on one H100 80GB HBM3 (400 W power limit), fp32, tol 1e-4, scale 1.05: pose graphs |Ax+g|/|g| <= 1.0e-4
    (bounds 2.0e-4 .. 1.3e-3), |x-x*|/|x*| <= 2.0e-3 (bounds 0.36 .. 16); bundle adjustment 5.6e-5 (bounds
    3.9e-4 .. 9.2e-3) and 4.6e-4 (bounds 29 .. 1e5).  The error bound is loose because lambda_min is bounded by the
    least-constrained unknown (a point seen twice, or a node at the end of the chain); the residual bound is the tight
    check.  fp64, tol 1e-13, scale 1 + 1e-4: |Ax+g|/|g| <= 1.0e-13, max-norm error <= 5.7e-10 (pose graphs) and
    2.1e-11 (bundle adjustment)."""
    u, xs = UNIT_ROUNDOFF[dt], x if xref is None else xref
    gn, xn = np.linalg.norm(g), np.linalg.norm(xs)
    kappa = abs(A).sum(1).max() * xn / gn
    res_bound = tol + 100 * u * kappa
    res = np.linalg.norm(A @ x + g) / gn
    msg = f"{tag}: |Ax+g|/|g| {res:.2e} (bound {res_bound:.2e})"
    assert res <= res_bound, msg
    if xref is not None:
        lam = (A.diagonal() - H.diagonal())[H.diagonal() > 0].min()
        err_bound = res_bound * gn / (lam * xn)
        err = np.linalg.norm(x - xref) / xn
        msg += f", |x-x*|/|x*| {err:.2e} (bound {err_bound:.2e})"
        assert err <= err_bound, msg
        if dt == torch.float64:
            assert np.abs(x - xref).max() <= errtol * np.abs(xref).max(), msg
    print(msg)


@pytest.mark.parametrize("N", PGO_N)
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_pgo_device_pcg_vs_sparse_solve(dtn, N):
    """Pose graph (chain + 300 banded loop closures) through both single-GPU routes, b200_lm_pgo2_pcg (node-ordered
    gathers) and b200_lm_pgo_pcg (per-edge scatter), against an fp64 sparse solve of (H + clamp/damp) x = -g.  fp64: error
    <= 1e-8 where the sparse LU is cheap (N <= 4500), predicted reduction to 1e-9; both dtypes: the bounds of _check_pcg,
    and the atomic-free route is bit-reproducible."""
    from pypose_b200.optim import _fused as F
    dt, scale, tol = PCG_DT[dtn]
    dmin, dmax, maxiter = 1e-6, 1e32, 20_000
    rng = np.random.default_rng(22)
    gt, init, edges, Z = _pgo_problem(rng, N, min(N, 300), meas_noise=0.02, span=30)
    ei, ej = (torch.from_numpy(edges[:, k].astype(np.int32)).cuda() for k in (0, 1))
    M, u, c = ops.lm_pgo_linearize(cu(init, dt), cu(Z, dt), ei, ej, 0, 1.0)
    Hd, g = ops.lm_pgo_scatter(M, u, ei, ej, N)
    # node-ordered copies and the gathered block sums (no atomics) must agree with the scatter kernel
    keys = torch.cat([ei, ej]).long()
    order = torch.sort(keys, stable=True)[1]
    nother = torch.cat([ej, ei])[order].contiguous()
    nptr = torch.zeros(N + 1, dtype=torch.int32, device="cuda")
    nptr[1:] = torch.cumsum(torch.bincount(keys, minlength=N), 0).to(torch.int32)
    pos = torch.empty(2 * len(ei), dtype=torch.int32, device="cuda")
    pos[order] = torch.arange(2 * len(ei), dtype=torch.int32, device="cuda")
    class _P:                                 # the attributes pgo_linearize_nodes reads from a PGOProblem
        pass
    prob = _P()
    prob.ei, prob.ej, prob.Z, prob.nptr = ei, ej, cu(Z, dt), nptr
    prob.epos_i, prob.epos_j = pos[:len(ei)].contiguous(), pos[len(ei):].contiguous()
    Mn, Hd_n, g_n, c_n = F.pgo_linearize_nodes("pgo", prob, cu(init, dt), 0, 1.0)
    lt = 1e-10 if dt == torch.float64 else 1e-5          # fp32: the atomics of the scatter kernel sum in another order
    assert (Hd_n - Hd).abs().max().item() <= lt * Hd.abs().max().item()
    assert (g_n - g).abs().max().item() <= lt * max(1.0, g.abs().max().item())
    assert abs(float(c_n[0]) - float(c[0])) <= lt * 1e-2 * float(c[0])
    H = _pgo_sparse_H(M.double().cpu().numpy(), edges, N)
    A = _damped(H, scale, dmin, dmax)
    gv = g.double().cpu().numpy().reshape(-1)
    xref = _ref_solve(A, -gv, N <= 4500) if N <= 4500 or dt == torch.float32 else None
    x, iters, pred = F.pgo_solve_nodes(Mn, nother, nptr, Hd_n, g_n, scale, dmin, dmax, tol, maxiter)   # gather, 2 kernels / it
    xr, itr, predr = F.pgo_solve_nodes(Mn, nother, nptr, Hd_n, g_n, scale, dmin, dmax, tol, maxiter)
    assert torch.equal(x, xr) and itr == iters and torch.equal(pred, predr)                            # bit-reproducible
    xs, iters_s, pred_s = F.pgo_solve(M, ei, ej, Hd, g, scale, dmin, dmax, tol, maxiter)               # scatter operator
    for route, xd, it, pr in (("pgo2", x, iters, pred), ("scatter", xs, iters_s, pred_s)):
        assert 0 < it < maxiter, (route, it)
        xv = xd.double().cpu().numpy().reshape(-1)
        _check_pcg(f"pgo {route} {dtn} N={N} iters={it}", H, A, gv, xv, xref, scale, tol, dt, 1e-8)
        if dt == torch.float64:
            np.testing.assert_allclose(pr.cpu().numpy()[0], xv @ (H @ xv) + 2 * xv @ gv, rtol=1e-9)


def _ba_geom(cidx, pidx, pix_t, C, P, split, tpi):
    """The BAProblem geometry for camera-sorted observations (numpy index arrays, device pixel tensor)."""
    padj = torch.from_numpy(np.argsort(pidx, kind="stable")).cuda()
    ppos = torch.empty(len(pidx), dtype=torch.int32, device="cuda")
    ppos[padj] = torch.arange(len(pidx), dtype=torch.int32, device="cuda")
    pptr = torch.from_numpy(np.concatenate([[0], np.cumsum(np.bincount(pidx, minlength=P))]).astype(np.int32)).cuda()
    cseg = torch.from_numpy(np.concatenate([[0], np.cumsum(np.bincount(cidx, minlength=C))]).astype(np.int32)).cuda()
    ci = torch.from_numpy(cidx.astype(np.int32)).cuda()
    return (cseg, split, tpi, ppos, ci[padj].contiguous(), pptr, pix_t[padj].contiguous()), padj


# (cameras, points, (items per camera S, threads per item) or None for what BAProblem picks, robust kind, delta, holes):
# every layout on a small problem; the single-CTA kernels <512> / <1024> and the grid path (each point seen by 3
# consecutive cameras); a few cameras with 2e5 rows (S = 21 items per camera) where camera 4 and point 5 have no observation
BA_CASES = ([(12, 150, lay, k, d, False) for lay in ((1, 32), (1, 128), (3, 32), (2, 128)) for k, d in ((0, 1.0), (1, 0.02))]
            + [(C, 5 * C, None, 0, 1.0, False) for C in (2500, 3500, 4500)]
            + [(9, 75_000, None, 0, 1.0, True)])


@pytest.mark.parametrize("C,P,layout,kind,delta,holes", BA_CASES,
                         ids=[f"C{c[0]}-{'x'.join(map(str, c[2])) if c[2] else 'auto'}-k{c[3]}{'-holes' if c[5] else ''}"
                              for c in BA_CASES])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_ba_device_schur_pcg_vs_sparse_solve(dtn, C, P, layout, kind, delta, holes):
    """b200_lm_ba_linearize_seg / point_blocks / schur_diag_seg / ba_pcg (csrc/ba.cu, no atomics) against the stored-row
    kernels, the oracle and an fp64 sparse solve of the full damped normal equations (cameras and points); two runs are
    bit-identical.  fp64: the item layout's camera blocks, gradients and Schur diagonal match the stored rows to 1e-9,
    the solution the sparse solve to 1e-7 (a gauge-free system), the back-substitution
    xp = -Hpp^-1 (gp + W^T xc) of the returned xc to 1e-10; both dtypes: the bounds of _check_pcg."""
    from pypose_b200.optim import _fused as F
    from pypose_b200.optim.structured import BAProblem
    dt, scale, tol = PCG_DT[dtn]
    dmin, dmax, maxiter = 1e-6, 1e32, 20_000
    f64 = dt == torch.float64
    rng = np.random.default_rng(23)
    gt, ptsw, T0, p0, pix, cidx, pidx = _ba_problem(rng, C, P, 3, pix_noise=0.01, consecutive=True)
    if holes:
        keep = (cidx != 4) & (pidx != 5)
        pix, cidx, pidx = pix[keep], cidx[keep], pidx[keep]
    o = np.argsort(cidx, kind="stable")
    pix, cidx, pidx = pix[o], cidx[o], pidx[o]
    m = len(cidx)
    Td, pd, xd = cu(T0, dt), cu(p0, dt), cu(pix, dt)
    ci, pi_ = torch.from_numpy(cidx.astype(np.int32)).cuda(), torch.from_numpy(pidx.astype(np.int32)).cuda()
    Jc, Jp, rs, Hcc, Hpp, gc, gp, cur = ops.lm_ba_linearize(Td, pd, xd, ci, pi_, kind, delta)
    if f64:
        outs_o = L.ba_linearize(T0, p0, pix, cidx, pidx, kind, delta)
        for a, b in zip((Jc, Jp, rs, Hcc, Hpp, gc, gp), outs_o):
            assert np.abs(a.cpu().numpy() - b).max() <= 1e-9 * max(1.0, np.abs(b).max())
    if layout is None:
        prob = BAProblem(pp.module.BundleAdjustment(pp.SE3(Td), pd), xd, ci, pi_, None, None, (kind, delta), tol, maxiter)
        split, tpi = prob.geom[1:3]
    else:
        split, tpi = layout
    assert split > 3 or not holes
    geom, padj = _ba_geom(cidx, pidx, xd, C, P, split, tpi)
    Y4s, rs_y, Hcc_y, Hpp_y, gc_y, gp_y, cur_y = F.ba_linearize_det(Td, pd, xd, pi_, geom, kind, delta)
    assert torch.equal(Y4s[1], Y4s[0][padj])
    if f64:
        for a, b in ((rs_y, rs), (Hcc_y, Hcc), (Hpp_y, Hpp), (gc_y, gc), (gp_y, gp), (cur_y, cur)):
            assert (a - b).abs().max().item() <= 1e-9 * max(1.0, b.abs().max().item())
        # Schur diagonal of the item layout (S partial sums per camera, folded in order) against the stored rows
        Hc, Hpinv = torch.empty(C, 21, dtype=dt, device="cuda"), torch.empty(P, 6, dtype=dt, device="cuda")
        F._launch("b200_lm_blk6_damp_inv", Hc, [F._p(Hcc_y), scale, dmin, dmax, F._p(Hc), None, None], C)
        F._launch("b200_lm_pt3_damp_inv", Hc, [F._p(Hpp_y), scale, dmin, dmax, F._p(Hpinv)], P)
        Sd = Hc.clone()
        part = torch.empty(C * split, 21, dtype=dt, device="cuda") if split > 1 else None
        F._launch("b200_lm_ba_schur_diag_seg", Hc, [F._p(Y4s[0]), F._p(Td), F._p(pi_), F._p(geom[0]), split, tpi, F._p(Hpinv),
                                                   F._p(Sd), F._p(part)], C)
        Jcn, Jpn = Jc.cpu().numpy().reshape(m, 2, 6), Jp.cpu().numpy().reshape(m, 2, 3)
        G = Jpn @ _dense_sym(Hpinv.cpu().numpy(), P, 3)[pidx] @ Jpn.transpose(0, 2, 1)
        S_ref = _dense_sym(Hc.cpu().numpy(), C, 6)
        np.subtract.at(S_ref, cidx, Jcn.transpose(0, 2, 1) @ G @ Jcn)
        assert np.abs(_dense_sym(Sd.cpu().numpy(), C, 6) - S_ref).max() <= 1e-9 * np.abs(S_ref).max()
    # both runs take every input from ba_linearize_det (rs of the stored-row kernel agrees with rs_y to rounding only)
    xc, xp, iters, pred = F.ba_solve(Y4s, Td, rs_y, ci, pi_, geom, Hcc_y, Hpp_y, gc_y, gp_y, scale, dmin, dmax, tol, maxiter)
    again = F.ba_linearize_det(Td, pd, xd, pi_, geom, kind, delta)
    xc2, xp2, iters2, pred2 = F.ba_solve(again[0], Td, again[1], ci, pi_, geom, *again[2:6], scale, dmin, dmax, tol, maxiter)
    assert torch.equal(xc, xc2) and torch.equal(xp, xp2) and iters == iters2 and torch.equal(pred, pred2)   # bit-reproducible
    assert 0 < iters < maxiter
    J = _ba_sparse_J(Jc.double().cpu().numpy(), Jp.double().cpu().numpy(), cidx, pidx, C, P)
    R = rs.double().cpu().numpy().reshape(-1)
    H = (J.T @ J).tocsr()
    A = _damped(H, scale, dmin, dmax)
    gv = J.T @ R
    got = np.concatenate([xc.double().cpu().numpy().reshape(-1), xp.double().cpu().numpy().reshape(-1)])
    _check_pcg(f"ba {dtn} C={C} S={split} tpi={tpi} iters={iters}", H, A, gv, got, _ba_ref_solve(A, -gv, C), scale, tol,
               dt, 1e-7)
    if f64:
        Jd = J @ got
        np.testing.assert_allclose(pred.cpu().numpy()[0], Jd @ (2 * R + Jd), rtol=1e-9)
        Hp = _dense_sym(Hpp.cpu().numpy(), P, 3)
        dp = np.einsum('pii->pi', Hp).copy()
        Hp[:, np.arange(3), np.arange(3)] = np.clip(dp, dmin, dmax) * scale
        rhs = gp.cpu().numpy() + L.ba_wtx(Jcn, Jpn, cidx, pidx, xc.cpu().numpy(), P)
        xp_ref = -np.linalg.solve(Hp, rhs[..., None])[..., 0]
        assert np.abs(xp.cpu().numpy() - xp_ref).max() <= 1e-10 * np.abs(xp_ref).max()
        y = ops.lm_ba_wv(Jc, Jp, ci, pi_, torch.ones(P, 3, dtype=dt, device="cuda"), C).cpu().numpy()
        np.testing.assert_allclose(y, L.ba_wv(outs_o[0], outs_o[1], cidx, pidx, np.ones((P, 3)), C), rtol=1e-9, atol=1e-9)


CG_RR, CG_DONE, CG_ITERS, CG_PATIENCE = 3, 5, 6, 11          # slots of the PCG state (csrc/pcg.cu)


def _pgo_pcg_by_iteration(M, ei, ej, Hd, g, scale, tol, maxiter, patience=None):
    """b200_lm_pgo_pcg enqueued one iteration per call (first_iter = k, iters = 1), the calls _fused.pgo_solve makes in
    chunks, then b200_lm_cg_finish.  Returns the iterates x_0 = 0, x_1, ... (copied after every call), |r_k|^2 from
    the state for k = 0, 1, ..., the state after the last call and the x that cg_finish leaves.  `patience`, if given,
    replaces the stagnation patience after the first call."""
    from pypose_b200.optim import _fused as F
    dev, dt, n, E = M.device, M.dtype, Hd.shape[0], M.shape[0]
    ws, cg = F._workspace(dev), F._cg(dev)
    extra, Minv = torch.empty(n, 6, dtype=dt, device=dev), torch.empty(n, 21, dtype=dt, device=dev)
    F._launch("b200_lm_blk6_damp_inv", M, [F._p(Hd), float(scale), 1e-6, 1e32, None, F._p(extra), F._p(Minv)], n)
    x, r, z, p, q, xbest = (torch.empty(n, 6, dtype=dt, device=dev) for _ in range(6))
    xs, rr = [torch.zeros_like(x)], [float((g.double() ** 2).sum())]
    for k in range(maxiter):
        F._launch("b200_lm_pgo_pcg", M, [F._p(M), F._p(ei), F._p(ej), E, F._p(Minv), F._p(extra), F._p(g), F._p(x), F._p(r),
                                         F._p(z), F._p(p), F._p(q), F._p(xbest), F._p(cg), F._p(ws), float(tol), maxiter, k, 1,
                                         *F._NOCOMM], n)
        st = cg.tolist()
        if st[CG_ITERS] == k + 1:
            xs.append(x.clone())
            rr.append(st[CG_RR])
        if k == 0 and patience is not None:
            cg[CG_PATIENCE] = patience
        if st[CG_DONE] != 0.0:
            break
    F._launch("b200_lm_cg_finish", M, [F._p(x), F._p(xbest), F._p(cg)], n)
    return xs, np.array(rr), st, x


@pytest.mark.parametrize("N", [90, 4500])                  # cg_vec_small_kernel<256>, grid path (cg_update)
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_pcg_guard_stop_reasons_return_the_best_iterate(dtn, N):
    """The PCG guard (DESIGN §3 "PCG guard"): the solve stops as converged (1), breakdown (2), stagnated (3) or maxiter (4)
    and returns the last iterate if it converged or if the last iterate has the smallest |r|, else the iterate with the
    smallest |r|.  The residual 2-norm of PCG is not monotone, so a solve stopped after an iteration where |r| rose
    must return an earlier iterate."""
    dt = PCG_DT[dtn][0]
    rng = np.random.default_rng(24)
    gt, init, edges, Z = _pgo_problem(rng, N, min(N, 300), meas_noise=0.02, span=30)
    ei, ej = (torch.from_numpy(edges[:, k].astype(np.int32)).cuda() for k in (0, 1))
    M, u, _ = ops.lm_pgo_linearize(cu(init, dt), cu(Z, dt), ei, ej, 0, 1.0)
    Hd, g = ops.lm_pgo_scatter(M, u, ei, ej, N)
    run = lambda tol, maxiter, **kw: _pgo_pcg_by_iteration(M, ei, ej, Hd, g, 1.0 + 1e-3, tol, maxiter, **kw)
    # converged: x is the last iterate
    xs, rr, st, x = run(1e-4, 20_000)
    assert st[CG_DONE] == 1.0 and st[CG_ITERS] == len(xs) - 1 and torch.equal(x, xs[-1])
    # maxiter, on a run that cannot converge: after 3 iterations; after an iteration where |r| rose; after one where it
    # reached a new minimum.  maxiter is honoured exactly and the returned iterate decreases the quadratic model.
    xs, rr, st, x = run(1e-30, 300)
    prior = np.minimum.accumulate(rr)
    rose = next(k for k in range(2, len(rr)) if rr[k] > 1.01 * prior[k - 1])
    fell = next(k for k in range(rose + 1, len(rr)) if rr[k] < 0.99 * prior[k - 1])
    A = _damped(_pgo_sparse_H(M.double().cpu().numpy(), edges, N), 1.0 + 1e-3, 1e-6, 1e32)
    gv = g.double().cpu().numpy().reshape(-1)
    for K in (3, rose, fell):
        xs, rr, st, x = run(1e-30, K)
        best = int(np.argmin(rr))
        assert st[CG_DONE] == 4.0 and st[CG_ITERS] == K and len(rr) == K + 1
        if K != 3:
            assert (best < K) == (K == rose), (K, best, rr)
        assert torch.equal(x, xs[best])
        xv = x.double().cpu().numpy().reshape(-1)
        assert xv @ (A @ xv) + 2 * xv @ gv < 0
    # stagnated: with the patience lowered to 2, the solve stops 2 iterations after its last new minimum of |r| (at N = 4500
    # the first two iterations in a row without a new minimum come after ~300)
    xs, rr, st, x = run(1e-30, 3000, patience=2.0)
    stop, since = None, 0
    for k in range(1, len(rr)):
        since = 0 if rr[k] < rr[:k].min() else since + 1
        if since >= 2:
            stop = k
            break
    assert stop is not None and st[CG_DONE] == 3.0 and st[CG_ITERS] == stop == len(rr) - 1
    assert torch.equal(x, xs[int(np.argmin(rr))])
    # breakdown: edge blocks -M (an indefinite operator; Hd still sets an SPD preconditioner) stop the first iteration
    xs, rr, st, x = _pgo_pcg_by_iteration(-M, ei, ej, Hd, g, 1.0 + 1e-3, 1e-4, 100)
    assert st[CG_DONE] == 2.0 and st[CG_ITERS] == 0.0 and len(xs) == 1
    assert torch.equal(x, torch.zeros_like(x))


def _smoke_ba(dev, dtype=torch.float32, tol=1e-6):
    """The bundle-adjustment block of smoke() (gauge-free, 6 cameras, fp32, PCG tolerance below what fp32 reaches)."""
    torch.manual_seed(0)
    Cb, Pb, per = 6, 80, 3
    gtb = pp.se3(0.2 * torch.randn(Cb, 6, device=dev, dtype=dtype)).Exp()
    ptw = (torch.rand(Pb, 3, device=dev, dtype=dtype) * torch.tensor([4.0, 4.0, 3.0], device=dev, dtype=dtype)
           + torch.tensor([-2.0, -2.0, 3.0], device=dev, dtype=dtype))
    pidx = torch.arange(Pb, device=dev).repeat_interleave(per)
    cidx = (pidx + torch.arange(per, device=dev).repeat(Pb) * 2) % Cb
    yb = gtb[cidx].Act(ptw[pidx])
    ba = pp.module.BundleAdjustment(pp.se3(0.02 * torch.randn(Cb, 6, device=dev, dtype=dtype)).Exp() * gtb,
                                    ptw + 0.03 * torch.randn(Pb, 3, device=dev, dtype=dtype))
    opt = pp.optim.LM(ba, solver=pp.optim.solver.PCG(tol=tol), sparse=True)
    inp = (-yb[:, :2] / yb[:, 2:], cidx, pidx)
    losses = [float(opt.step(inp)) for _ in range(3)]
    return losses, ba.poses.tensor().clone(), ba.points_3d.detach().clone()


def test_smoke_bundle_adjustment_is_reproducible_and_converges():
    """The smoke() BA scenario once gave a different outcome on every run (atomics + fp32 CG run past its attainable
    accuracy).  Now: 20 runs are bit-identical and every one meets smoke()'s bound."""
    ref = _smoke_ba("cuda")
    l0, l1 = ref[0][0], ref[0][1]
    assert l1 < 0.1 * l0 + 1e-8, ref[0]
    for _ in range(19):
        got = _smoke_ba("cuda")
        assert got[0] == ref[0] and torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2])


def test_pgo_weighted_kernels_vs_oracle():
    rng = np.random.default_rng(31)
    gt, init, edges, Z = _pgo_problem(rng, 300, 250, meas_noise=0.02)
    E = len(edges)
    B = rng.standard_normal((E, 6, 6))
    W = B @ B.transpose(0, 2, 1) / 6 + 0.5 * np.eye(6)
    ei, ej = (torch.from_numpy(edges[:, k].astype(np.int32)).cuda() for k in (0, 1))
    for dt, tol in ((torch.float64, 1e-9), (torch.float32, 2e-4)):
        for Wc in (W, W[:1]):
            for kind, delta in ((0, 1.0), (1, 0.1)):
                outs = ops.lm_pgo_linearize_w(cu(init, dt), cu(Z, dt), ei, ej, cu(Wc, dt), kind, delta)
                outs_o = L.pgo_linearize(cu(init, dt).double().cpu().numpy(), cu(Z, dt).double().cpu().numpy(), edges[:, 0],
                                         edges[:, 1], kind, delta, W=cu(Wc, dt).double().cpu().numpy())
                for a, b, nm in zip(outs, outs_o, ("M", "u", "M0", "u0", "cost")):
                    assert np.abs(a.double().cpu().numpy() - b).max() <= tol * max(1.0, np.abs(b).max()), (nm, dt)
    # predicted reduction from per-edge blocks
    from pypose_b200.optim import _fused as F
    D = cu(rng.standard_normal((300, 6)), torch.float64)
    M0, u0 = outs[2].double(), outs[3].double()
    ws = F._workspace(D.device)
    F._launch("b200_lm_pgo_predicted_edge", M0, [F._p(M0), F._p(u0), F._p(ei), F._p(ej), F._p(D), F._p(ws)], E)
    d = (D[ej.long()] - D[ei.long()]).cpu().numpy()
    Mb = _dense_sym(M0.cpu().numpy(), E, 6)
    ref = np.einsum('ei,eij,ej->', d, Mb, d) + 2 * (d * u0.cpu().numpy()).sum()
    np.testing.assert_allclose(ws[0].item(), ref, rtol=1e-10)


@pytest.mark.parametrize("case", ["trustregion", "constant", "shared"])
def test_lm_pgo_information_matrices_reference_trajectory_on_gpu(golden_lm, case):
    g = golden_lm
    W = torch.from_numpy(g["pgo_w/infos"].copy()).cuda()
    W = W[3] if case == "shared" else W
    st = pp.optim.strategy.Constant(damping=1e-4) if case == "constant" else pp.optim.strategy.TrustRegion()
    net = pp.module.PoseGraph(pp.SE3(torch.from_numpy(g["pgo/nodes0"].copy()).cuda()))
    inp = (torch.from_numpy(g["pgo/edges"]).cuda(), pp.SE3(torch.from_numpy(g["pgo/Z"].copy()).cuda()))
    opt = pp.optim.LM(net, strategy=st, solver=pp.optim.solver.PCG(tol=1e-13), sparse=True)
    for k in range(5):
        loss = opt.step(inp, weight=W)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g[f"pgo_w/{case}/loss"][k], rtol=1e-6)
        np.testing.assert_allclose(net.nodes.detach().cpu().numpy(), g[f"pgo_w/{case}/poses"][k],
                                   atol=2e-7 if not (case == "shared" and k >= 3) else 2e-5)   # see docstring / note below
        assert opt.reject_count == g[f"pgo_w/{case}/reject"][k]


def test_reference_sparse_lm_scenarios_gpu():
    """tests/optim/test_sparse_lm.py of the reference (identity model with a target; chain pose graph with a fixed root)."""
    from tests.test_lm import run_sparse_lm_scenarios
    run_sparse_lm_scenarios(torch.device("cuda"))


def test_gauss_newton_structured_route_on_gpu_at_scale():
    """GN on 1e4 poses / 1e6 reprojection residuals (the reference's dense pinv would need a 2e6 x 7e4 matrix)."""
    rng = np.random.default_rng(41)
    gt, init, pts, pix, cidx = _reproj_problem(rng, 10_000, 1_000_000, noise=0.03)
    net = pp.module.PoseReproj(pp.SE3(cu(init, torch.float32)))
    inp = (cu(pts, torch.float32), cu(pix, torch.float32), torch.from_numpy(cidx).cuda())
    opt = pp.optim.GN(net)
    losses = [float(opt.step(inp)) for _ in range(5)]
    assert opt._problem is not None
    assert losses[-1] < 1e-6 * losses[0] + 1e-4, losses


@pytest.mark.parametrize("route", ["gather", "scatter"])
def test_lm_pgo_gather_and_scatter_routes(golden_lm, route):
    """Unweighted: node-ordered gathers (csrc/pcg2.cu, no atomics) — reference trajectory and two bit-identical runs;
    identity information matrices: the per-edge scatter kernels (the weighted and multi-GPU operator) — same trajectory."""
    g = golden_lm
    W = torch.eye(6, dtype=torch.float64, device="cuda") if route == "scatter" else None
    finals = []
    for _ in range(2):
        net = pp.module.PoseGraph(pp.SE3(torch.from_numpy(g["pgo/nodes0"].copy()).cuda()))
        inp = (torch.from_numpy(g["pgo/edges"]).cuda(), pp.SE3(torch.from_numpy(g["pgo/Z"].copy()).cuda()))
        opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), solver=pp.optim.solver.PCG(tol=1e-12), sparse=True)
        for k in range(5):
            loss = opt.step(inp, weight=W)
            assert opt._problem is not None and (opt._problem.W is None) == (route == "gather")
            assert (getattr(opt._problem, "_pds", None) is not None) == (route == "gather")     # native step driver (lmdrive.cu)
            np.testing.assert_allclose(float(loss), g["pgo/trustregion/loss"][k], rtol=1e-6)
            np.testing.assert_allclose(net.nodes.detach().cpu().numpy(), g["pgo/trustregion/poses"][k], atol=1e-7)
        finals.append(net.nodes.detach().clone())
    if route == "gather":
        assert torch.equal(finals[0], finals[1])


@pytest.mark.parametrize("kname,kern", [("huber", lambda: pp.optim.kernel.Huber(delta=0.1)),
                                        ("cauchy", lambda: pp.optim.kernel.Cauchy(delta=0.2))])
def test_lm_pgo_robust_kernels_reference_trajectory_on_gpu(golden_lm, kname, kern):
    g = golden_lm
    net = pp.module.PoseGraph(pp.SE3(torch.from_numpy(g["pgo/nodes0"].copy()).cuda()))
    inp = (torch.from_numpy(g["pgo/edges"]).cuda(), pp.SE3(torch.from_numpy(g["pgo_robust/Z"].copy()).cuda()))
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), kernel=kern(), solver=pp.optim.solver.PCG(tol=1e-13), sparse=True)
    for k in range(5):
        loss = opt.step(inp)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g[f"pgo_robust/{kname}/loss"][k], rtol=1e-6)
        np.testing.assert_allclose(net.nodes.detach().cpu().numpy(), g[f"pgo_robust/{kname}/poses"][k], atol=5e-7)
        assert opt.reject_count == g[f"pgo_robust/{kname}/reject"][k]


def test_lm_bundle_adjustment_huber_reference_trajectory_on_gpu(golden_lm):
    g = golden_lm
    net = pp.module.BundleAdjustment(pp.SE3(torch.from_numpy(g["ba/poses0"].copy()).cuda()),
                                     torch.from_numpy(g["ba/points0"].copy()).cuda())
    inp = (torch.from_numpy(g["ba_robust/pix"].copy()).cuda(), torch.from_numpy(g["ba/cidx"]).cuda(), torch.from_numpy(g["ba/pidx"]).cuda())
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), kernel=pp.optim.kernel.Huber(delta=0.05),
                      solver=pp.optim.solver.PCG(tol=1e-13), sparse=True)
    for k in range(5):
        loss = opt.step(inp)
        assert opt._problem is not None
        np.testing.assert_allclose(float(loss), g["ba_robust/huber/loss"][k], rtol=1e-5)
        np.testing.assert_allclose(net.poses.detach().cpu().numpy(), g["ba_robust/huber/poses"][k], atol=2e-6)
        np.testing.assert_allclose(net.points_3d.detach().cpu().numpy(), g["ba_robust/huber/points"][k], atol=2e-6)
        assert opt.reject_count == g["ba_robust/huber/reject"][k]


# ------------------------------------------------------------------ two-pose reprojection (config 5 as stated)
def test_reproj2_kernels_vs_oracle():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "lm2.npz"))
    nodes, pts, ia, ib = g["poses0"], g["pts"], g["ia"], g["ib"]
    N = nodes.shape[0]
    order = np.argsort(ia * N + ib, kind="stable")
    key = (ia * N + ib)[order]
    uniq, counts = np.unique(key, return_counts=True)
    pa, pb = (uniq // N).astype(np.int32), (uniq % N).astype(np.int32)
    pseg = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    for tag, intr in (("readme", L.README_INTR), ("k", (320.0, 0.5, 310.0, 300.0, 250.0))):
        pix = g["pix_k"] if tag == "k" else g["pix_readme"]
        for dt, tol in ((torch.float64, 1e-10), (torch.float32, 3e-5)):
            for kind, delta in ((0, 1.0), (1, 0.5 if tag == "k" else 0.002)):
                M, u, c = ops.lm_reproj2_accum(cu(nodes, dt), cu(pts[order], dt), cu(pix[order], dt), torch.from_numpy(pseg).cuda(),
                                               torch.from_numpy(pa).cuda(), torch.from_numpy(pb).cuda(), list(intr), kind, delta)
                Mo, uo, co = L.reproj2_accum(cu(nodes, dt).double().cpu().numpy(), cu(pts[order], dt).double().cpu().numpy(),
                                             cu(pix[order], dt).double().cpu().numpy(), pseg, pa, pb, intr, kind, delta)
                for a, b, nm in ((M, Mo, "M"), (u, uo, "u"), (c, co, "cost")):
                    assert np.abs(a.double().cpu().numpy() - b).max() <= tol * max(1.0, np.abs(b).max()), (tag, dt, kind, nm)
                l = ops.lm_reproj2_loss(cu(nodes, dt), cu(pts[order], dt), cu(pix[order], dt), torch.from_numpy(pseg).cuda(),
                                        torch.from_numpy(pa).cuda(), torch.from_numpy(pb).cuda(), list(intr), kind, delta)
                assert abs(float(l[0]) - co[0]) <= tol * max(1.0, abs(co[0]))


@pytest.mark.parametrize("tag,strategy", [("readme", "trustregion"), ("readme", "constant"), ("k", "trustregion"), ("hard", "trustregion")])
def test_lm_two_pose_reprojection_matches_reference_trajectory_gpu(tag, strategy):
    from tests.test_lm import _lm2_run
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "lm2.npz"))
    steps = 8 if tag == "hard" else 6
    run = _lm2_run(g, tag, strategy, "structured", dev="cuda", steps=steps)
    ref_loss = g[f"{tag}/{strategy}/loss"]
    for k, (loss, poses, rej) in enumerate(run):
        np.testing.assert_allclose(loss, ref_loss[k], rtol=1e-5 if tag == "hard" else 2e-6)
        if tag != "hard":
            np.testing.assert_allclose(poses, g[f"{tag}/{strategy}/poses"][k], atol=2e-7)
        if k == 0 or ref_loss[k - 1] - ref_loss[k] > 1e-9 * ref_loss[k]:
            assert rej == g[f"{tag}/{strategy}/reject"][k]


def test_lm_two_pose_reprojection_fp32_converges_to_1e5():
    """north_star: LM converged pose error <= 1e-5, here in fp32 on the block-sparse config: noise-free pixels, so the
    relative poses T_b^-1 T_a of every observed pair must come back to ground truth (the absolute poses keep the gauge)."""
    rng = np.random.default_rng(3)
    N, per = 500, 24
    # a closed loop of radius 3 (several laps): fp32 resolves ~4e-7 at |t| = 3; on an open trajectory that wanders hundreds
    # of units from the origin the cancellation in R_b^T (w - t_b) alone exceeds 1e-5
    th = 0.05 * np.arange(N)
    rot = np.stack([np.zeros(N), np.zeros(N), th], 1) + 0.05 * rng.standard_normal((N, 3))
    gt = O.exp("SE3", np.concatenate([np.zeros((N, 3)), rot], 1))
    gt[:, :3] = np.stack([3 * np.cos(th), 3 * np.sin(th), 0.3 * np.sin(3 * th)], 1)
    ia = np.repeat(np.arange(N - 3), 3 * per)
    ib = ia + np.tile(np.repeat([1, 2, 3], per), N - 3)
    m = len(ia)
    yb = rng.uniform([-2, -2, 2], [2, 2, 6], (m, 3))
    rel = O.mul("SE3", O.inv("SE3", gt[ia]), gt[ib])
    pts = O.act("SE3", rel, yb)
    pix = -yb[:, :2] / yb[:, 2:]
    init = O.mul("SE3", O.exp("SE3", 0.02 * rng.standard_normal((N, 6))), gt)
    net = pp.module.TwoPoseReproj(pp.SE3(cu(init, torch.float32)))
    opt = pp.optim.LM(net, solver=pp.optim.solver.PCG(tol=1e-5, maxiter=1000), sparse=True)
    inp = (cu(pts, torch.float32), cu(pix, torch.float32), torch.from_numpy(ia).cuda(), torch.from_numpy(ib).cuda())
    for _ in range(15):
        opt.step(inp)
    P = net.poses.detach().double().cpu().numpy()
    est = O.mul("SE3", O.inv("SE3", P[ib[::per]]), P[ia[::per]])
    ref = O.mul("SE3", O.inv("SE3", gt[ib[::per]]), gt[ia[::per]])
    err = np.abs(O.log("SE3", O.mul("SE3", O.inv("SE3", ref), est))).max()
    assert err <= 1e-5, err


@pytest.mark.parametrize("declare", [True, False])
def test_generic_block_route_matches_reference_dense_run_gpu(declare):
    """The generic block route (sjac / psjac, optim/blocks.py) on CUDA: Jacobian blocks through the op-level backward
    kernels, trajectory of the reference's dense LM (oracle/make_golden_lm2.py "bak"); then the same model at 1e6 residual
    rows, which the dense route cannot hold (J would be 2e6 x 3.8e5)."""
    from tests.test_lm import BAWithIntrinsics
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "lm.npz"))
    g2 = np.load(os.path.join(os.path.dirname(__file__), "golden", "lm2.npz"))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    net = BAWithIntrinsics(pp.SE3(t(g["ba/poses0"])), t(g["ba/points0"]), t(g2["bak/K"]), declare).cuda()
    opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), solver=pp.optim.solver.PCG(tol=1e-12), sparse=True)
    inp = (t(g2["bak/pix"]), t(g["ba/cidx"]), t(g["ba/pidx"]))
    for k in range(5):
        loss = opt.step(inp)
        assert type(opt._problem).__name__ == "BlockProblem"
        np.testing.assert_allclose(float(loss), g2["bak/trustregion/loss"][k], rtol=1e-5)
        np.testing.assert_allclose(net.poses.detach().cpu().numpy(), g2["bak/trustregion/poses"][k], atol=1e-6)
    if not declare:
        return
    rng = np.random.default_rng(9)
    C, P = 1000, 125_000
    gt, ptsw, T0, p0, pix, cidx, pidx = _ba_problem(rng, C, P, 8, pix_noise=0.0)
    K = torch.tensor([[-1.2, 0.01, 0.05], [0.0, -0.9, -0.02], [0.0, 0.0, 1.0]], device="cuda")
    ci_t, pi_t = torch.from_numpy(cidx).cuda(), torch.from_numpy(pidx).cuda()
    pixk = pp.point2pixel(pp.SE3(cu(gt, torch.float32))[ci_t].Act(cu(ptsw, torch.float32)[pi_t]), K)     # exact pixels
    big = BAWithIntrinsics(pp.SE3(cu(T0, torch.float32)), cu(p0, torch.float32), K, True).cuda()
    opt = pp.optim.LM(big, solver=pp.optim.solver.PCG(tol=1e-3, maxiter=40), sparse=True)
    inp = (pixk, ci_t, pi_t)
    losses = [float(opt.step(inp)) for _ in range(4)]
    assert type(opt._problem).__name__ == "BlockProblem" and len(cidx) == 1_000_000
    assert losses[-1] < 1e-3 * losses[0], losses
