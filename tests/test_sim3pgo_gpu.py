"""Sim3 pose graphs on the GPU (csrc/sim3pgo.cu, the width-7 kernels of csrc/pcg2.cu / pcg.cu, the family-2 trial of
csrc/lmdrive.cu, optim/structured.py Sim3PGOProblem) against the fp64 oracle (oracle/sim3pgo_oracle.py) and the reference's
dense LM trajectories (tests/golden/sim3pgo.npz), in fp64 and fp32."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch
from torch import nn

import pypose_b200 as pp
from oracle import lie_oracle as L
from oracle import sim3pgo_oracle as S
from pypose_b200.optim import _fused, structured
from pypose_b200.optim.solver import PCG

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sim3pgo.npz")
TOL = {torch.float64: 1e-9, torch.float32: 5e-4}


def cu(a, dt=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max(initial=0.0) / (1.0 + np.abs(b).max(initial=0.0))


def golden_case(name):
    g = np.load(GOLDEN)
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


class UserPoseGraph(nn.Module):
    """examples/module/pgo `PoseGraph` as a user writes it."""

    def __init__(self, nodes):
        super().__init__()
        self.nodes = pp.Parameter(nodes)

    def forward(self, edges, poses):
        node1 = self.nodes[edges[..., 0]]
        node2 = self.nodes[edges[..., 1]]
        return (poses.Inv() @ node1.Inv() @ node2).Log().tensor()


def edge_cases():
    """A drift graph plus: an isolated node, a hub whose degree is far above the 4 lanes per node, an edge with r = 0 and
    theta = 0 (identity rotations, Z = A^-1 B exactly), scales exactly 1 and scales from 0.2 to 5."""
    d = S.problem(11, N=16, loops=4)
    nodes, edges, Z = d["nodes0"].copy(), d["edges"], d["Z"]
    N = len(nodes)
    rng = np.random.default_rng(3)
    nodes[:, 7] = np.geomspace(0.2, 5.0, N)
    nodes[0, 7] = 1.0
    extra = np.zeros((3, 8))
    extra[:, 6] = extra[:, 7] = 1.0
    extra[1, :3] = [0.5, -0.2, 0.1]
    extra[2, :3] = [1.0, 0.3, -0.4]
    nodes = np.concatenate([nodes, extra])               # N: isolated, N+1, N+2: identity rotations, unit scale
    hub = N + 1
    more = [(hub, k) for k in range(0, N, 1)] + [(N + 1, N + 2)]
    Zm = []
    for i, j in more:
        rel_ = L.mul("Sim3", L.inv("Sim3", nodes[i]), nodes[j])
        if (i, j) == (N + 1, N + 2):
            Zm.append(rel_)                                 # r = 0, theta = 0
        else:
            Zm.append(L.mul("Sim3", rel_, L.exp("Sim3", rng.normal(0, 0.05, 7))))
    edges = np.concatenate([edges, np.array(more, np.int64)])
    Z = np.concatenate([Z, np.stack(Zm)])
    return nodes, edges, Z


def problem_on_gpu(nodes, edges, Z, dt, robust=(0, 1.0)):
    model = pp.module.PoseGraph(pp.Sim3(cu(nodes, dt))).cuda()
    prob = structured.Sim3PGOProblem(model, torch.from_numpy(edges).cuda(), pp.Sim3(cu(Z, dt)), None, robust, 1e-12, None)
    return model, prob


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
@pytest.mark.parametrize("kind,delta", [(0, 1.0), (1, 0.05), (3, 0.3)])
def test_linearize_node_sums_and_loss_match_oracle(dt, kind, delta):
    nodes, edges, Z = edge_cases()
    N = len(nodes)
    _, prob = problem_on_gpu(nodes, edges, Z, dt, (kind, delta))
    x = prob._nodes().detach()
    Mn, Hd, g, cur = _fused.pgo_linearize_nodes("sim3", prob, x, kind, delta)
    # the oracle at the nodes the kernels saw (fp32 inputs rounded)
    nd, Zd = x.double().cpu().numpy(), prob.Z.double().cpu().numpy()
    b = S.blocks(nd, Zd, edges, kind, delta)
    Mo, uo, (epos_i, epos_j, nptr, nother) = S.node_blocks(b, edges, N)
    np.testing.assert_array_equal(prob.epos_i.cpu().numpy(), epos_i)
    np.testing.assert_array_equal(prob.nptr.cpu().numpy(), nptr)
    assert rel(Mn.cpu().numpy(), Mo) < TOL[dt]
    Hdo, go = S.node_sums(b, edges, N)
    assert rel(Hd.cpu().numpy(), S.pack(Hdo)) < TOL[dt]
    assert rel(g.cpu().numpy(), go) < TOL[dt]
    iso = N - 3                                                          # the isolated node (edge_cases)
    np.testing.assert_array_equal(Hd[iso].cpu().numpy(), 0.0)
    np.testing.assert_array_equal(g[iso].cpu().numpy(), 0.0)
    assert abs(float(cur[0]) - b["loss"]) <= TOL[dt] * (1 + b["loss"])
    loss = float(_fused.sim3pgo_loss(x, prob.Z, prob.ei, prob.ej, kind, delta)[0])
    assert abs(loss - b["loss"]) <= TOL[dt] * (1 + b["loss"])
    # the edge with r = 0 and theta = 0 and the scales from 0.2 to 5 give finite blocks
    assert torch.isfinite(Mn).all() and torch.isfinite(g).all()
    # no atomics: a second launch is bit-identical
    Mn2, Hd2, g2, cur2 = _fused.pgo_linearize_nodes("sim3", prob, x, kind, delta)
    assert torch.equal(Mn, Mn2) and torch.equal(Hd, Hd2) and torch.equal(g, g2) and torch.equal(cur, cur2)


def _dense(Hd, Mn, nptr, nother, N):
    """scipy sparse H from the node-ordered blocks (off-diagonal -M at every slot)."""
    iu = np.triu_indices(7)
    def unpack(p):
        A = np.zeros((7, 7))
        A[iu] = p
        return A + np.triu(A, 1).T
    rows, cols, vals = [], [], []
    for n in range(N):
        blk = [(n, unpack(Hd[n]))] + [(nother[s], -unpack(Mn[s])) for s in range(nptr[n], nptr[n + 1])]
        for m, A in blk:
            r, c = np.meshgrid(7 * n + np.arange(7), 7 * m + np.arange(7), indexing="ij")
            rows.append(r.ravel()); cols.append(c.ravel()); vals.append(A.ravel())
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(7 * N, 7 * N))


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
def test_damp_pcg_and_predicted_match_scipy(dt):
    nodes, edges, Z = edge_cases()
    N = len(nodes)
    _, prob = problem_on_gpu(nodes, edges, Z, dt)
    Mn, Hd, g, _ = _fused.pgo_linearize_nodes("sim3", prob, prob._nodes(), 0, 1.0)
    H = _dense(Hd.double().cpu().numpy(), Mn.double().cpu().numpy(), prob.nptr.cpu().numpy(), prob.nother.cpu().numpy(), N)
    assert abs(H - H.T).max() < 1e-12 * abs(H).max()
    scale = 1.3
    # clamp + damp + inverse of the 7x7 blocks
    Hdo = np.stack([H[7 * n:7 * n + 7, 7 * n:7 * n + 7].toarray() for n in range(N)])
    Hdamp, extra_o = S.damp(Hdo, scale)
    Hdd, extra, Minv = torch.empty_like(Hd), torch.empty_like(g), torch.empty_like(Hd)
    _fused._launch("b200_lm_sim3pgo_damp_inv", Hd, [Hd.data_ptr(), scale, 1e-6, 1e32, Hdd.data_ptr(), extra.data_ptr(),
                                                    Minv.data_ptr()], N)
    assert rel(Hdd.cpu().numpy(), S.pack(Hdamp)) < TOL[dt]
    assert rel(extra.cpu().numpy(), extra_o) < TOL[dt]
    assert rel(Minv.cpu().numpy(), S.pack(np.linalg.inv(Hdamp))) < (1e-8 if dt == torch.float64 else 1e-3)
    # PCG against spsolve on the damped system
    A = (H + sp.diags(extra.double().cpu().numpy().reshape(-1))).tocsc()
    ref = spla.spsolve(A, -g.double().cpu().numpy().reshape(-1)).reshape(N, 7)
    x, iters, pred = _fused.pgo_solve_nodes(Mn, prob.nother, prob.nptr, Hd, g, scale, 1e-6, 1e32,
                                            1e-12 if dt == torch.float64 else 1e-6, None)
    assert 0 < iters <= 70 * N
    assert rel(x.cpu().numpy(), ref) < (1e-8 if dt == torch.float64 else 2e-3)
    # predicted reduction (operator in mode 1) at the solution and at a random step
    for xv in (x, torch.randn_like(x)):
        xn = xv.double().cpu().numpy().reshape(-1)
        want = xn @ (H @ xn) + 2 * xn @ g.double().cpu().numpy().reshape(-1)
        ws = _fused._workspace(x.device)
        _fused._launch("b200_lm_sim3pgo_predicted", Mn, [Mn.data_ptr(), prob.nother.data_ptr(), prob.nptr.data_ptr(),
                                                         xv.data_ptr(), g.data_ptr(), ws.data_ptr()], N)
        assert abs(float(ws[0]) - want) <= TOL[dt] * (1 + abs(want) + abs(xn @ (abs(H) @ abs(xn))))


CASES = {"constant": (pp.optim.strategy.Constant, 0, 1.0), "trustregion": (pp.optim.strategy.TrustRegion, 0, 1.0),
         "reject": (pp.optim.strategy.TrustRegion, 0, 1.0), "huber": (pp.optim.strategy.TrustRegion, 1, 0.05),
         "module": (pp.optim.strategy.TrustRegion, 0, 1.0)}


def _run(name, device_step, monkeypatch, dt=torch.float64):
    g = golden_case(name)
    cls, rk, delta = CASES[name]
    strategy = cls(damping=1e-6) if cls is pp.optim.strategy.Constant else cls()
    nodes = pp.Sim3(cu(g["nodes0"], dt))
    model = UserPoseGraph(nodes) if name == "module" else pp.module.PoseGraph(nodes)
    kernel = pp.optim.kernel.Huber(delta=delta) if rk == 1 else None
    if not device_step:
        monkeypatch.setattr(structured.Sim3PGOProblem, "device_step", lambda self, s: None)
    opt = pp.optim.LM(model, strategy=strategy, kernel=kernel, solver=PCG(tol=1e-13), sparse=True, reject=16)
    inp = (torch.from_numpy(g["edges"]).cuda(), pp.Sim3(cu(g["Z"], dt)))
    loss, out, rej = [], [], []
    for _ in range(len(g["loss"])):
        loss.append(float(opt.step(input=inp)))
        out.append(model.nodes.detach().tensor().double().cpu().numpy())
        rej.append(opt.reject_count)
    assert isinstance(opt._problem, structured.Sim3PGOProblem)
    assert (getattr(opt._problem, "_pds", None) is not None) == device_step        # one C call per trial
    return g, np.array(loss), np.stack(out), np.array(rej)


@pytest.mark.parametrize("device_step", [True, False])
@pytest.mark.parametrize("case", sorted(CASES))
def test_trajectory_matches_reference_dense_lm(case, device_step, monkeypatch):
    g, loss, nodes, rej = _run(case, device_step, monkeypatch)
    np.testing.assert_array_equal(rej, g["reject"])
    np.testing.assert_allclose(loss, g["loss"], rtol=1e-6)
    np.testing.assert_allclose(nodes, g["nodes"], rtol=0, atol=1e-6)


def test_repeat_runs_are_bit_identical(monkeypatch):
    a = _run("reject", True, monkeypatch, torch.float32)
    b = _run("reject", True, monkeypatch, torch.float32)
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[2], b[2])


def test_fused_route_agrees_with_generic_route(monkeypatch):
    g = golden_case("trustregion")
    inp = (torch.from_numpy(g["edges"]).cuda(), pp.Sim3(cu(g["Z"])))
    out = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setattr(structured, "recognize", lambda *a, **k: None)
        model = pp.module.PoseGraph(pp.Sim3(cu(g["nodes0"])))
        opt = pp.optim.LM(model, strategy=pp.optim.strategy.TrustRegion(), solver=PCG(tol=1e-13), sparse=True)
        losses = [float(opt.step(input=inp)) for _ in range(3)]
        assert isinstance(opt._problem, structured.Sim3PGOProblem) == fused
        out.append((np.array(losses), model.nodes.detach().tensor().cpu().numpy()))
    np.testing.assert_allclose(out[0][0], out[1][0], rtol=1e-6)
    np.testing.assert_allclose(out[0][1], out[1][1], rtol=0, atol=1e-6)


def test_fp32_large_graph_converges():
    torch.manual_seed(0)
    N, dev = 100_000, torch.device("cuda")
    steps = torch.zeros(N, 7, device=dev, dtype=torch.float64)
    steps[1:, 0] = 1.0
    steps[1:, 3:6] = 0.05 * torch.randn(N - 1, 3, device=dev, dtype=torch.float64)
    gt = pp.sim3(steps).Exp().cumprod(dim=0, left=False)
    chain = torch.stack([torch.arange(N - 1), torch.arange(1, N)], 1)
    a = torch.randint(0, N - 20, (2 * N,))
    loops = torch.stack([a, a + torch.randint(2, 20, (2 * N,))], 1)
    edges = torch.cat([chain, loops]).to(dev)
    Z = pp.Sim3((gt[edges[:, 0]].Inv() @ gt[edges[:, 1]]).tensor().float())
    start = (pp.sim3(0.02 * torch.randn(N, 7, device=dev, dtype=torch.float64)).Exp() @ gt).tensor().float()
    model = pp.module.PoseGraph(pp.Sim3(start.clone()))
    opt = pp.optim.LM(model, strategy=pp.optim.strategy.TrustRegion(), solver=PCG(tol=1e-6), sparse=True)
    losses = [float(opt.step(input=(edges, Z))) for _ in range(4)]
    prob = opt._problem
    assert isinstance(prob, structured.Sim3PGOProblem) and prob._pds is not None
    first = float(_fused.sim3pgo_loss(start, prob.Z, prob.ei, prob.ej)[0])
    assert all(np.isfinite(losses)) and losses[-1] < 1e-3 * first, (first, losses)


def _problem_of(model, inp, **kw):
    opt = pp.optim.LM(model, **kw)
    try:
        opt.step(input=inp)
    except Exception:                        # a fall-through route may not support the input; only the route matters
        pass
    return opt._problem


def test_other_inputs_keep_their_routes():
    g = golden_case("constant")
    e = torch.from_numpy(g["edges"])
    kw = dict(solver=PCG(), sparse=True)
    # information matrices, mixed dtypes, CPU tensors, GaussNewton: not the Sim3 route
    m = pp.module.PoseGraph(pp.Sim3(cu(g["nodes0"])))
    W = torch.eye(7, dtype=torch.float64, device="cuda").expand(len(e), 7, 7)
    assert not isinstance(_problem_of(m, (e.cuda(), pp.Sim3(cu(g["Z"]))), weight=W, **kw), structured.Sim3PGOProblem)
    m = pp.module.PoseGraph(pp.Sim3(cu(g["nodes0"])))
    assert not isinstance(_problem_of(m, (e.cuda(), pp.Sim3(cu(g["Z"], torch.float32))), **kw), structured.Sim3PGOProblem)
    m = pp.module.PoseGraph(pp.Sim3(torch.from_numpy(g["nodes0"])))
    assert structured.recognize(m, (e, pp.Sim3(torch.from_numpy(g["Z"]))), list(m.parameters()), solver=PCG(), sparse=True) is None
    m = pp.module.PoseGraph(pp.Sim3(cu(g["nodes0"])))
    gn = pp.optim.GaussNewton(m)
    gn.step(input=(e.cuda(), pp.Sim3(cu(g["Z"]))))
    assert gn._problem is None
    # a process group, and no iterative solver asked for
    inp = (e.cuda(), pp.Sim3(cu(g["Z"])))
    assert structured.recognize(m, inp, list(m.parameters()), group=True, solver=PCG(), sparse=True) is None
    assert structured.recognize(m, inp, list(m.parameters())) is None
    # RxSO3 / SO3 graphs
    for grp, rnd in ((pp.RxSO3, pp.randn_RxSO3), (pp.SO3, pp.randn_SO3)):
        m = pp.module.PoseGraph(rnd(12, dtype=torch.float64, device="cuda"))
        Zr = rnd(len(e), dtype=torch.float64, device="cuda")
        assert structured.recognize(m, (e.cuda(), Zr), list(m.parameters()), solver=PCG(), sparse=True) is None
    # SE3 graphs still take the SE3 problem class
    m = pp.module.PoseGraph(pp.randn_SE3(12, dtype=torch.float64, device="cuda"))
    prob = structured.recognize(m, (e.cuda(), pp.randn_SE3(len(e), dtype=torch.float64, device="cuda")), list(m.parameters()),
                                solver=PCG(), sparse=True)
    assert type(prob) is structured.PGOProblem
    # a user module whose residual differs is not recognised
    class Other(UserPoseGraph):
        def forward(self, edges, poses):
            return 2.0 * super().forward(edges, poses)
    m = Other(pp.Sim3(cu(g["nodes0"])))
    assert structured.recognize(m, inp, list(m.parameters()), solver=PCG(), sparse=True) is None
