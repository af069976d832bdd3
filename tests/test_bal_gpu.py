"""BAL bundle adjustment on the GPU (csrc/bal.cu, optim/structured.py BALProblem) against the fp64 oracle
(oracle/bal_oracle.py) and the reference's dense LM trajectories (tests/golden/bal.npz), in fp64 and fp32."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch
from torch import nn

import pypose_b200 as pp
from oracle import bal_oracle as B
from pypose_b200.autograd.function import psjac
from pypose_b200.optim import _fused, structured
from pypose_b200.optim.solver import PCG

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IU = np.triu_indices(9)
IU3 = np.triu_indices(3)


def cu(a, dt=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max(initial=0.0) / (1.0 + np.abs(b).max(initial=0.0))


def with_unobserved(d):
    """One extra camera and one extra point without observations."""
    d = dict(d)
    d["K0"] = np.concatenate([d["K0"], d["K0"][:1]])
    d["T0"] = np.concatenate([d["T0"], d["T0"][:1]])
    d["P0"] = np.concatenate([d["P0"], d["P0"][:1] + 0.1])
    return d


class Layout:
    """BALProblem's observation layout with a chosen (split, tpi)."""

    def __init__(self, d, dt, split=None, tpi=None):
        self.dtype = dt
        C, P = len(d["K0"]), len(d["P0"])
        structured._group_by_camera(self, cu(d["pix"], dt), torch.from_numpy(d["cidx"]).cuda(),
                                    torch.from_numpy(d["pidx"]).cuda(), C, P)
        g = list(self.geom)
        if split is not None:
            g[1], g[2] = split, tpi
        self.geom = tuple(g)
        self.order = np.argsort(d["cidx"], kind="stable")


def sorted_oracle(d, kind=0, delta=1.0):
    o = np.argsort(d["cidx"], kind="stable")
    ci, pi_, pix = d["cidx"][o], d["pidx"][o], d["pix"][o]
    return B.blocks(d["K0"], d["T0"], d["P0"], pix, ci, pi_, kind, delta), ci, pi_


GEOMS = [(1, 32), (1, 128), (3, 32), (4, 128)]


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("kind", [(0, 1.0), (1, 20.0), (3, 20.0)])
def test_linearize_blocks_match_oracle(dt, geom, kind):
    d = with_unobserved(B.problem(5, C=6, P=50, M=600))
    lay = Layout(d, dt, *geom)
    K, T, P = cu(d["K0"], dt), cu(d["T0"], dt), cu(d["P0"], dt)
    (Y4, Y4p), rs, Hcc, Hpp, gc, gp, cur = _fused.bal_linearize(K, T, P, lay.pix, lay.pidx, lay.geom, *kind)
    b, _, _ = sorted_oracle(d, *kind)
    tol = 1e-10 if dt == torch.float64 else 2e-4
    assert rel(Hcc.cpu(), b["Hcc"][:, IU[0], IU[1]]) < tol
    assert rel(gc.cpu(), b["gc"]) < tol
    assert rel(Hpp.cpu(), b["Hpp"][:, IU3[0], IU3[1]]) < tol
    assert rel(gp.cpu(), b["gp"]) < tol
    assert rel(rs.cpu(), b["rs"]) < tol
    assert abs(float(cur) - b["loss"]) <= tol * (1 + b["loss"])
    assert float(Hcc[-1].abs().max()) == 0.0 and float(Hpp[-1].abs().max()) == 0.0      # unobserved camera / point


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
@pytest.mark.parametrize("geom", [(1, 32), (3, 128)])
def test_schur_products_predicted_and_trial_loss_match_oracle(dt, geom):
    d = with_unobserved(B.problem(6, C=6, P=50, M=600))
    lay = Layout(d, dt, *geom)
    K, T, P = cu(d["K0"], dt), cu(d["T0"], dt), cu(d["P0"], dt)
    Y4s, rs, Hcc, Hpp, gc, gp, cur = _fused.bal_linearize(K, T, P, lay.pix, lay.pidx, lay.geom)
    b, ci, pi_ = sorted_oracle(d)
    C, Pn, scale = len(d["K0"]), len(d["P0"]), 1.3
    S, rhs, Sd, Hpinv = B.schur(b, ci, pi_, scale)
    cseg, split, tpi, _, cidx_p, pptr, _ = lay.geom
    Y4, Y4p = Y4s
    seg = [_fused._p(Y4), _fused._p(T), _fused._p(K), _fused._p(lay.pidx), _fused._p(cseg), split, tpi]
    part = torch.empty(C * split, 45, dtype=dt, device="cuda") if split > 1 else None
    Hc = torch.empty(C, 45, dtype=dt, device="cuda")
    Hpi = torch.empty(Pn, 6, dtype=dt, device="cuda")
    _fused._launch("b200_lm_bal_damp_inv", Y4, [_fused._p(Hcc), scale, 1e-6, 1e32, _fused._p(Hc), None], C)
    _fused._launch("b200_lm_pt3_damp_inv", Y4, [_fused._p(Hpp), scale, 1e-6, 1e32, _fused._p(Hpi)], Pn)
    Sdg = Hc.clone()
    _fused._launch("b200_lm_bal_schur_diag_seg", Y4, [*seg, _fused._p(Hpi), _fused._p(Sdg), _fused._p(part)], C)
    tol = 1e-9 if dt == torch.float64 else 2e-3
    # the kernel sums W_k Hpp^-1 W_k^T per observation: the Schur diagonal block when every (camera, point) pair is
    # observed once (BAL files); with repeated pairs, as in these random problems, it omits their cross terms
    Wk = np.swapaxes(b["Jc"], 1, 2) @ b["Jp"]
    Sd_obs = B.damp(b["Hcc"], scale, 1e-6, 1e32)
    np.add.at(Sd_obs, ci, -(Wk @ Hpinv[pi_] @ np.swapaxes(Wk, 1, 2)))
    assert rel(Sdg.cpu(), Sd_obs[:, IU[0], IU[1]]) < tol
    # W v and W^T x against the oracle's products
    rng = np.random.default_rng(1)
    t, x = rng.normal(size=(Pn, 3)), rng.normal(size=(C, 9))
    y = torch.zeros(C, 9, dtype=dt, device="cuda")
    _fused._launch("b200_lm_bal_wv_seg", Y4, [*seg, None, _fused._p(cu(t, dt)), _fused._p(y), _fused._p(part)], C)
    assert rel(y.cpu(), -B.wv(b["Jc"], b["Jp"], ci, pi_, t, C)) < tol
    u = torch.empty(Pn, 3, dtype=dt, device="cuda")
    _fused._launch("b200_lm_bal_wtx_gather", Y4, [_fused._p(Y4p), _fused._p(T), _fused._p(K), _fused._p(cidx_p),
                                                  _fused._p(pptr), _fused._p(Hpi), _fused._p(cu(x, dt)), None, 1.0,
                                                  _fused._p(u)], Pn)
    ref = np.einsum("jab,jb->ja", Hpinv, B.wtx(b["Jc"], b["Jp"], ci, pi_, x, Pn))
    assert rel(u.cpu(), ref) < tol
    # the whole solve (tight PCG), the predicted reduction and the trial loss
    xc, xp, iters, pred = _fused.bal_solve(Y4s, K, T, rs, lay.cidx, lay.pidx, lay.geom, Hcc, Hpp, gc, gp, scale, 1e-6,
                                           1e32, 1e-12 if dt == torch.float64 else 1e-6, 500)
    xc0, xp0, pred0 = B.dense_step(b, ci, pi_, scale)
    stol = 1e-7 if dt == torch.float64 else 5e-2
    assert rel(xc.cpu(), xc0) < stol and rel(xp.cpu(), xp0) < stol
    assert abs(float(pred) - pred0) <= stol * abs(pred0)
    Kt, Tt, Pt = _fused.bal_retract(K, T, P, xc, xp)
    K1, T1, P1 = B.retract(d["K0"], d["T0"], d["P0"], xc.cpu().double().numpy(), xp.cpu().double().numpy())
    assert rel(Kt.cpu(), K1) < tol and rel(Tt.cpu(), T1) < tol and rel(Pt.cpu(), P1) < tol
    tl = _fused.bal_loss(Kt, Tt, Pt, lay.pix, lay.cidx, lay.pidx)
    ref_tl = B.blocks(K1, T1, P1, d["pix"], d["cidx"], d["pidx"])["loss"]
    assert abs(float(tl) - ref_tl) <= (1e-9 if dt == torch.float64 else 1e-4) * ref_tl


def scipy_reduced_solve(b, ci, pi_, scale):
    """Damped reduced camera system S = Hc - W Hpp^-1 W^T solved by scipy's CG on sparse W (block-Jacobi preconditioned
    with the exact diagonal blocks, tolerance far below the GPU solve's)."""
    C, Pn = len(b["gc"]), len(b["gp"])
    Hc = B.damp(b["Hcc"], scale, 1e-6, 1e32)
    Hpinv = np.linalg.inv(B.damp(b["Hpp"], scale, 1e-6, 1e32))
    Wk = np.swapaxes(b["Jc"], 1, 2) @ b["Jp"]
    rr = (9 * ci[:, None, None] + np.arange(9)[None, :, None]).repeat(3, 2)
    cc = (3 * pi_[:, None, None] + np.arange(3)[None, None, :]).repeat(9, 1)
    W = sp.csr_matrix((Wk.ravel(), (rr.ravel(), cc.ravel())), shape=(9 * C, 3 * Pn))
    Hpi, Hcd = sp.block_diag(list(Hpinv), format="csr"), sp.block_diag(list(Hc), format="csr")
    S = spla.LinearOperator((9 * C, 9 * C), matvec=lambda x: Hcd @ x - W @ (Hpi @ (W.T @ x)), dtype=np.float64)
    Sd = Hc.copy()
    np.add.at(Sd, ci, -(Wk @ Hpinv[pi_] @ np.swapaxes(Wk, 1, 2)))
    Minv = sp.block_diag(list(np.linalg.inv(Sd)), format="csr")
    rhs = -b["gc"].reshape(-1) + W @ (Hpi @ b["gp"].reshape(-1))
    x, info = spla.cg(S, rhs, rtol=1e-13, atol=0.0, maxiter=20000, M=Minv)
    assert info == 0
    return x.reshape(-1, 9)


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
# cg_vec_small_kernel<256> (C <= 2048), cg_vec_small_kernel<512> (2048 < C <= kVecSmallRows = 4096), the grid path (C > 4096)
@pytest.mark.parametrize("C", [300, 3000, 5000])
def test_pcg_solution_matches_scipy(dt, C):
    d = B.problem(7, C=C, P=2 * C, M=8 * C)
    lay = Layout(d, dt)
    K, T, P = cu(d["K0"], dt), cu(d["T0"], dt), cu(d["P0"], dt)
    Y4s, rs, Hcc, Hpp, gc, gp, cur = _fused.bal_linearize(K, T, P, lay.pix, lay.pidx, lay.geom)
    b, ci, pi_ = sorted_oracle(d)
    scale = 1.5
    xc, xp, iters, pred = _fused.bal_solve(Y4s, K, T, rs, lay.cidx, lay.pidx, lay.geom, Hcc, Hpp, gc, gp, scale, 1e-6,
                                           1e32, 1e-10 if dt == torch.float64 else 1e-5, 2000)
    x0 = scipy_reduced_solve(b, ci, pi_, scale)
    assert rel(xc.cpu(), x0) < (1e-6 if dt == torch.float64 else 5e-2), iters


# ---- trajectories against the reference's dense LM ---------------------------------------------------------------
class Reproj(nn.Module):                   # examples/module/ba/bundle_adjustment.py, unchanged
    def __init__(self, K, C, P):
        super().__init__()
        self.K = pp.Parameter(K, sjac=True)
        self.C = pp.Parameter(C, sjac=True)
        self.P = pp.Parameter(P, sjac=True)

    def forward(self, observe, cidx, pidx):
        return Reproj.project(self.K[cidx], self.C[cidx], self.P[pidx]) - observe

    @psjac
    def project(K, C, P):
        cp = C.Act(P)
        n = - cp[..., :2] / cp[..., [2]]
        radius = n.square().sum(dim=-1, keepdim=True)
        focal, k1, k2 = K[..., :1], K[..., 1:2], K[..., 2:3]
        distortion = 1 + k1 * radius + k2 * radius.square()
        return focal * distortion * n


class ReprojPlain(Reproj):                 # the same model without @psjac
    def forward(self, observe, cidx, pidx):
        return ReprojPlain.project(self.K[cidx], self.C[cidx], self.P[pidx]) - observe

    @staticmethod
    def project(K, C, P):
        cp = C.Act(P)
        n = - cp[..., :2] / cp[..., [2]]
        radius = n.square().sum(dim=-1, keepdim=True)
        return K[..., :1] * (1 + K[..., 1:2] * radius + K[..., 2:3] * radius.square()) * n


def golden_case(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", "bal.npz"))
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


def make(kind, K, T, P, dt=torch.float64):
    K, T, P = cu(K, dt), pp.SE3(cu(T, dt)), cu(P, dt)
    return {"module": lambda: pp.module.BALBundleAdjustment(K, T, P), "reproj": lambda: Reproj(K, T, P),
            "plain": lambda: ReprojPlain(K, T, P)}[kind]()


def params_of(model):
    if isinstance(model, pp.module.BALBundleAdjustment):
        return model.intrinsics, model.poses, model.points_3d
    return model.K, model.C, model.P


STRATS = {"constant": lambda: pp.optim.strategy.Constant(damping=1e-6), "trustregion": pp.optim.strategy.TrustRegion,
          "reject": pp.optim.strategy.TrustRegion}


@pytest.mark.parametrize("case", sorted(STRATS))
@pytest.mark.parametrize("kind", ["module", "reproj", "plain"])
def test_trajectory_matches_reference_dense_lm(case, kind):
    g = golden_case(case)
    model = make(kind, g["K0"], g["T0"], g["P0"])
    inp = (cu(g["pix"]), torch.from_numpy(g["cidx"]).cuda(), torch.from_numpy(g["pidx"]).cuda())
    opt = pp.optim.LM(model, solver=PCG(tol=1e-12, maxiter=2000), strategy=STRATS[case](), reject=16, sparse=True)
    for s in range(len(g["loss"])):
        loss = float(opt.step(inp))
        assert type(opt._problem).__name__ == "BALProblem"
        K, T, P = (t.detach().cpu().numpy() for t in params_of(model))
        assert opt.reject_count == g["reject"][s], s
        assert abs(loss - g["loss"][s]) <= 1e-5 * g["loss"][s], (s, loss, g["loss"][s])
        q, qg = T[:, 3:], g["T"][s][:, 3:]
        sign = np.sign((q * qg).sum(1, keepdims=True))
        assert np.abs(T[:, :3] - g["T"][s][:, :3]).max() < 1e-6 and np.abs(q * sign - qg).max() < 1e-6, s
        assert np.abs(P - g["P"][s]).max() < 1e-6, s
        ktol = 1e-4 if case == "reject" else 1e-6      # from the far start k2 is weakly determined by the first steps
        assert (np.abs(K - g["K"][s]) / np.maximum(np.abs(g["K"][s]), 1e-3)).max() < ktol, s


def test_fused_route_agrees_with_generic_route():
    d = B.problem(8, C=6, P=40, M=300, scale=2.0)
    inp = (cu(d["pix"]), torch.from_numpy(d["cidx"]).cuda(), torch.from_numpy(d["pidx"]).cuda())
    runs = []
    for generic in (False, True):
        model = make("module", d["K0"], d["T0"], d["P0"])
        opt = pp.optim.LM(model, solver=PCG(tol=1e-12, maxiter=2000), strategy=pp.optim.strategy.Constant(damping=1e-4),
                          sparse=True)
        if generic:               # the block route the same model takes when it is not recognised
            from pypose_b200.optim import blocks
            params = [p for p in model.parameters() if p.requires_grad]
            opt._problem = blocks.BlockProblem.build(model, inp, params, structured._input_key(inp), None, None,
                                                     opt.solver, opt.model)
            assert type(opt._problem).__name__ == "BlockProblem"
        losses = [float(opt.step(inp)) for _ in range(3)]
        runs.append((losses, [t.detach().cpu().numpy() for t in params_of(model)]))
    (la, pa), (lb, pb) = runs
    np.testing.assert_allclose(la, lb, rtol=1e-6)
    for a, b in zip(pa, pb):
        assert rel(a, b) < 1e-6


def synthetic(C, P, M, seed, dt):
    d = B.problem(seed, C=C, P=P, M=M, noise=0.01)        # a noise floor far below the starting loss
    return d, (cu(d["pix"], dt), torch.from_numpy(d["cidx"]).cuda(), torch.from_numpy(d["pidx"]).cuda())


def test_fp32_large_problem_converges_and_is_bit_reproducible():
    d, inp = synthetic(300, 40000, 400000, 9, torch.float32)
    out = []
    for _ in range(2):
        model = make("module", d["K0"], d["T0"], d["P0"], torch.float32)
        opt = pp.optim.LM(model, solver=PCG(tol=1e-4, maxiter=250), strategy=pp.optim.strategy.TrustRegion(), sparse=True)
        l0 = float(model(*inp).double().square().sum())
        for _ in range(10):
            loss = float(opt.step(inp))
        assert type(opt._problem).__name__ == "BALProblem"
        assert l0 / loss > 1e3, (l0, loss)
        out.append([t.detach().clone() for t in params_of(model)])
    for a, b in zip(*out):
        assert torch.equal(a, b)


# ---- recognition negatives: these keep the routes they take without BALProblem ----------------------------------
class NoK2(Reproj):
    def forward(self, observe, cidx, pidx):
        K, C, P = self.K[cidx], self.C[cidx], self.P[pidx]
        cp = C.Act(P)
        n = - cp[..., :2] / cp[..., [2]]
        radius = n.square().sum(dim=-1, keepdim=True)
        return K[..., :1] * (1 + K[..., 1:2] * radius) * n - observe


@pytest.mark.parametrize("case", ["no_k2", "frozen_intrinsics", "cpu"])
def test_other_models_keep_their_routes_and_converge(case):
    """A residual without k2 and CPU tensors converge on their routes; frozen intrinsics are only checked for the route
    decision (LM over a module with a frozen parameter fails in the generic routes, with or without this family)."""
    d = B.problem(10, C=5, P=30, M=200)
    if case == "cpu":
        K, T, P = (torch.from_numpy(d[k]).double() for k in ("K0", "T0", "P0"))
        model = pp.module.BALBundleAdjustment(K, pp.SE3(T), P)
        inp = (torch.from_numpy(d["pix"]), torch.from_numpy(d["cidx"]), torch.from_numpy(d["pidx"]))
    else:
        cls = NoK2 if case == "no_k2" else Reproj
        model = cls(cu(d["K0"]), pp.SE3(cu(d["T0"])), cu(d["P0"]))
        if case == "frozen_intrinsics":
            model.K.requires_grad_(False)
        inp = (cu(d["pix"]), torch.from_numpy(d["cidx"]).cuda(), torch.from_numpy(d["pidx"]).cuda())
    if case == "frozen_intrinsics":       # two trainable parameters: not the BAL family
        params = [p for p in model.parameters() if p.requires_grad]
        prob = structured.recognize(model, inp, params, None, (0, 1.0), PCG(), True)
        assert prob is None or type(prob).__name__ != "BALProblem"
        return
    opt = pp.optim.LM(model, solver=PCG(tol=1e-8, maxiter=500), strategy=pp.optim.strategy.TrustRegion(), sparse=True)
    l0 = float(model(*inp).double().square().sum())
    for _ in range(5):
        loss = float(opt.step(inp))
    assert type(opt._problem).__name__ != "BALProblem"
    assert loss < l0
