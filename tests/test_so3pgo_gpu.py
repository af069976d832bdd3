"""SO3 pose graphs (rotation averaging) on the GPU (csrc/so3pgo.cu, the width-3 kernels of csrc/pcg2.cu / pcg.cu, the
family-3 trial of csrc/lmdrive.cu, optim/structured.py SO3PGOProblem) against the fp64 oracle (oracle/so3pgo_oracle.py)
and the reference's dense LM trajectories (tests/golden/so3pgo.npz), in fp64 and fp32."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch
from torch import nn

import pypose_b200 as pp
from oracle import lie_oracle as L
from oracle import so3pgo_oracle as S
from pypose_b200.optim import _fused, structured
from pypose_b200.optim.solver import PCG

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "so3pgo.npz")
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
    """A view graph of 240 cameras plus: an isolated node, a hub joined to every camera (degree 240, far above the 4 lanes
    per node), an edge with r = 0 and theta = 0 (identity rotations, Z = identity) and an edge whose residual is
    pi - 1e-3.  Returns nodes, edges, Z and the index of the isolated node."""
    d = S.problem(11, N=240, deg=6)
    nodes, edges, Z = d["nodes0"], d["edges"], d["Z"]
    N = len(nodes)
    rng = np.random.default_rng(3)
    eye = np.array([0.0, 0.0, 0.0, 1.0])
    hub = L.exp("SO3", rng.normal(0, 1, 3))
    nodes = np.concatenate([nodes, np.stack([eye, hub, eye, eye])])   # N: isolated, N+1: hub, N+2, N+3: identity
    more = [(N + 1, k) for k in range(N)] + [(N + 2, N + 3), (0, 1)]
    Zm = []
    for i, j in more:
        rel_ = L.mul("SO3", L.inv("SO3", nodes[i]), nodes[j])
        if (i, j) == (N + 2, N + 3):
            Zm.append(rel_)                                 # r = 0, theta = 0
        elif (i, j) == (0, 1):                              # r = v, |v| = pi - 1e-3
            v = rng.normal(0, 1, 3)
            v *= (np.pi - 1e-3) / np.linalg.norm(v)
            Zm.append(L.mul("SO3", rel_, L.exp("SO3", -v)))
        else:
            Zm.append(L.mul("SO3", rel_, L.exp("SO3", rng.normal(0, 0.05, 3))))
    return nodes, np.concatenate([edges, np.array(more, np.int64)]), np.concatenate([Z, np.stack(Zm)]), N


def dense_graph():
    """A view graph with about 40 relative rotations per camera."""
    d = S.problem(12, N=80, deg=40, far=0.2)
    return d["nodes0"], d["edges"], d["Z"], None


GRAPHS = {"edge_cases": edge_cases, "dense": dense_graph}


def problem_on_gpu(nodes, edges, Z, dt, robust=(0, 1.0)):
    model = pp.module.PoseGraph(pp.SO3(cu(nodes, dt))).cuda()
    prob = structured.SO3PGOProblem(model, torch.from_numpy(edges).cuda(), pp.SO3(cu(Z, dt)), None, robust, 1e-12, None)
    return model, prob


@pytest.mark.parametrize("graph", sorted(GRAPHS))
@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
@pytest.mark.parametrize("kind,delta", [(0, 1.0), (1, 0.05), (3, 0.1)])
def test_linearize_node_sums_and_loss_match_oracle(dt, kind, delta, graph):
    nodes, edges, Z, iso = GRAPHS[graph]()
    N = len(nodes)
    _, prob = problem_on_gpu(nodes, edges, Z, dt, (kind, delta))
    x = prob._nodes().detach()
    Mn, Hd, g, cur = _fused.pgo_linearize_nodes("so3", prob, x, kind, delta)
    assert Mn.shape == (2 * len(edges), 8) and Hd.shape == (N, 6) and g.shape == (N, 3)
    # the oracle at the nodes the kernels saw (fp32 inputs rounded)
    nd, Zd = x.double().cpu().numpy(), prob.Z.double().cpu().numpy()
    b = S.blocks(nd, Zd, edges, kind, delta)
    Mo, uo, (epos_i, epos_j, nptr, nother) = S.node_blocks(b, edges, N)
    np.testing.assert_array_equal(prob.epos_i.cpu().numpy(), epos_i)
    np.testing.assert_array_equal(prob.nptr.cpu().numpy(), nptr)
    assert rel(Mn.cpu().numpy(), Mo) < TOL[dt]
    np.testing.assert_array_equal(Mn[:, 6:].cpu().numpy(), 0.0)          # slot padding
    Hdo, go = S.node_sums(b, edges, N)
    assert rel(Hd.cpu().numpy(), S.pack(Hdo)) < TOL[dt]
    assert rel(g.cpu().numpy(), go) < TOL[dt]
    if iso is not None:
        assert nptr[iso + 1] - nptr[iso] == 0 and nptr[iso + 2] - nptr[iso + 1] == iso
        np.testing.assert_array_equal(Hd[iso].cpu().numpy(), 0.0)
        np.testing.assert_array_equal(g[iso].cpu().numpy(), 0.0)
        assert np.abs(b["r"][-2]).max() == 0.0                           # the r = 0, theta = 0 edge
        assert abs(np.linalg.norm(b["r"][-1]) - (np.pi - 1e-3)) < (1e-9 if dt == torch.float64 else 1e-5)
    else:
        assert np.diff(nptr).mean() >= 39 and np.diff(nptr).min() >= 25
    assert abs(float(cur[0]) - b["loss"]) <= TOL[dt] * (1 + b["loss"])
    loss = float(_fused.so3pgo_loss(x, prob.Z, prob.ei, prob.ej, kind, delta)[0])
    assert abs(loss - b["loss"]) <= TOL[dt] * (1 + b["loss"])
    assert torch.isfinite(Mn).all() and torch.isfinite(g).all()
    # no atomics: a second launch is bit-identical
    Mn2, Hd2, g2, cur2 = _fused.pgo_linearize_nodes("so3", prob, x, kind, delta)
    assert torch.equal(Mn, Mn2) and torch.equal(Hd, Hd2) and torch.equal(g, g2) and torch.equal(cur, cur2)


def _dense(Hd, Mn, nptr, nother, N):
    """scipy sparse H from the node-ordered blocks (off-diagonal -M at every slot)."""
    iu = np.triu_indices(3)
    def unpack(p):
        A = np.zeros((3, 3))
        A[iu] = p[:6]
        return A + np.triu(A, 1).T
    rows, cols, vals = [], [], []
    for n in range(N):
        blk = [(n, unpack(Hd[n]))] + [(nother[s], -unpack(Mn[s])) for s in range(nptr[n], nptr[n + 1])]
        for m, A in blk:
            r, c = np.meshgrid(3 * n + np.arange(3), 3 * m + np.arange(3), indexing="ij")
            rows.append(r.ravel()); cols.append(c.ravel()); vals.append(A.ravel())
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * N, 3 * N))


@pytest.mark.parametrize("graph", sorted(GRAPHS))
@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
def test_damp_pcg_and_predicted_match_scipy(dt, graph):
    nodes, edges, Z, _ = GRAPHS[graph]()
    N = len(nodes)
    _, prob = problem_on_gpu(nodes, edges, Z, dt, (3, 0.1))
    Mn, Hd, g, _ = _fused.pgo_linearize_nodes("so3", prob, prob._nodes(), 3, 0.1)
    H = _dense(Hd.double().cpu().numpy(), Mn.double().cpu().numpy(), prob.nptr.cpu().numpy(), prob.nother.cpu().numpy(), N)
    assert abs(H - H.T).max() < 1e-12 * abs(H).max()
    scale = 1.3
    # clamp + damp + inverse of the 3x3 blocks
    Hdo = np.stack([H[3 * n:3 * n + 3, 3 * n:3 * n + 3].toarray() for n in range(N)])
    Hdamp, extra_o = S.damp(Hdo, scale)
    Hdd, extra, Minv = torch.empty_like(Hd), torch.empty_like(g), torch.empty_like(Hd)
    _fused._launch("b200_lm_so3pgo_damp_inv", Hd, [Hd.data_ptr(), scale, 1e-6, 1e32, Hdd.data_ptr(), extra.data_ptr(),
                                                   Minv.data_ptr()], N)
    assert rel(Hdd.cpu().numpy(), S.pack(Hdamp)) < TOL[dt]
    assert rel(extra.cpu().numpy(), extra_o) < TOL[dt]
    Mo = np.linalg.inv(Hdamp)
    assert np.abs(Minv.double().cpu().numpy() - S.pack(Mo)).max() <= (1e-8 if dt == torch.float64 else 1e-3) * (1 + np.abs(Mo).max())
    # PCG against spsolve on the damped system
    A = (H + sp.diags(extra.double().cpu().numpy().reshape(-1))).tocsc()
    ref = spla.spsolve(A, -g.double().cpu().numpy().reshape(-1)).reshape(N, 3)
    x, iters, pred = _fused.pgo_solve_nodes(Mn, prob.nother, prob.nptr, Hd, g, scale, 1e-6, 1e32,
                                            1e-12 if dt == torch.float64 else 1e-6, None)
    assert 0 < iters <= 30 * N
    assert rel(x.cpu().numpy(), ref) < (1e-8 if dt == torch.float64 else 2e-3)
    # predicted reduction (operator in mode 1) at the solution and at a random step
    for xv in (x, torch.randn_like(x)):
        xn = xv.double().cpu().numpy().reshape(-1)
        want = xn @ (H @ xn) + 2 * xn @ g.double().cpu().numpy().reshape(-1)
        ws = _fused._workspace(x.device)
        _fused._launch("b200_lm_so3pgo_predicted", Mn, [Mn.data_ptr(), prob.nother.data_ptr(), prob.nptr.data_ptr(),
                                                        xv.data_ptr(), g.data_ptr(), ws.data_ptr()], N)
        assert abs(float(ws[0]) - want) <= TOL[dt] * (1 + abs(want) + abs(xn @ (abs(H) @ abs(xn))))


CASES = {"constant": (pp.optim.strategy.Constant, None), "trustregion": (pp.optim.strategy.TrustRegion, None),
         "far": (pp.optim.strategy.TrustRegion, None), "huber": (pp.optim.strategy.TrustRegion, ("huber", 0.05)),
         "cauchy": (pp.optim.strategy.TrustRegion, ("cauchy", 0.1)), "module": (pp.optim.strategy.TrustRegion, None)}


def _run(name, device_step, monkeypatch, dt=torch.float64):
    g = golden_case(name)
    cls, k = CASES[name]
    strategy = cls(damping=1e-6) if cls is pp.optim.strategy.Constant else cls()
    nodes = pp.SO3(cu(g["nodes0"], dt))
    model = UserPoseGraph(nodes) if name == "module" else pp.module.PoseGraph(nodes)
    kernel = None if k is None else (pp.optim.kernel.Huber if k[0] == "huber" else pp.optim.kernel.Cauchy)(delta=k[1])
    if not device_step:
        monkeypatch.setattr(structured.SO3PGOProblem, "device_step", lambda self, s: None)
    opt = pp.optim.LM(model, strategy=strategy, kernel=kernel, solver=PCG(tol=1e-13), sparse=True, reject=16)
    inp = (torch.from_numpy(g["edges"]).cuda(), pp.SO3(cu(g["Z"], dt)))
    loss, out, rej = [], [], []
    for _ in range(len(g["loss"])):
        loss.append(float(opt.step(input=inp)))
        out.append(model.nodes.detach().tensor().double().cpu().numpy())
        rej.append(opt.reject_count)
    assert isinstance(opt._problem, structured.SO3PGOProblem)
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
    a = _run("far", True, monkeypatch, torch.float32)
    b = _run("far", True, monkeypatch, torch.float32)
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[2], b[2])


def test_fused_route_agrees_with_generic_route(monkeypatch):
    g = golden_case("cauchy")
    inp = (torch.from_numpy(g["edges"]).cuda(), pp.SO3(cu(g["Z"])))
    out = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setattr(structured, "recognize", lambda *a, **k: None)
            monkeypatch.setattr(structured, "recognize_so3_graph", lambda *a, **k: None)
        model = pp.module.PoseGraph(pp.SO3(cu(g["nodes0"])))
        opt = pp.optim.LM(model, strategy=pp.optim.strategy.TrustRegion(), kernel=pp.optim.kernel.Cauchy(delta=0.1),
                          solver=PCG(tol=1e-13), sparse=True)
        losses = [float(opt.step(input=inp)) for _ in range(3)]
        assert isinstance(opt._problem, structured.SO3PGOProblem) == fused
        out.append((np.array(losses), model.nodes.detach().tensor().cpu().numpy()))
    np.testing.assert_allclose(out[0][0], out[1][0], rtol=1e-6)
    np.testing.assert_allclose(out[0][1], out[1][1], rtol=0, atol=1e-6)


def test_fp32_large_graph_converges():
    torch.manual_seed(0)
    N, dev = 100_000, torch.device("cuda")
    gt = pp.randn_SO3(N, sigma=1.0, device=dev, dtype=torch.float64)
    chain = torch.stack([torch.arange(N - 1), torch.arange(1, N)], 1)
    a = torch.randint(0, N - 50, (4 * N,))
    loops = torch.stack([a, a + torch.randint(2, 50, (4 * N,))], 1)
    edges = torch.cat([chain, loops]).to(dev)
    Z = pp.SO3((gt[edges[:, 0]].Inv() @ gt[edges[:, 1]]).tensor().float())
    start = (pp.so3(0.1 * torch.randn(N, 3, device=dev, dtype=torch.float64)).Exp() @ gt).tensor().float()
    model = pp.module.PoseGraph(pp.SO3(start.clone()))
    opt = pp.optim.LM(model, strategy=pp.optim.strategy.TrustRegion(), solver=PCG(tol=1e-6), sparse=True)
    losses = [float(opt.step(input=(edges, Z))) for _ in range(4)]
    prob = opt._problem
    assert isinstance(prob, structured.SO3PGOProblem) and prob._pds is not None
    first = float(_fused.so3pgo_loss(start, prob.Z, prob.ei, prob.ej)[0])
    assert all(np.isfinite(losses)) and losses[-1] < 1e-3 * first, (first, losses)


def _problem_of(model, inp, **kw):
    opt = pp.optim.LM(model, **kw)
    try:
        opt.step(input=inp)
    except Exception:                        # a fall-through route may not support the input; only the route matters
        pass
    return opt._problem


def test_recognition():
    g = golden_case("constant")
    e = torch.from_numpy(g["edges"])
    kw = dict(solver=PCG(), sparse=True)
    inp = (e.cuda(), pp.SO3(cu(g["Z"])))
    rec = structured.recognize_so3_graph
    # the built-in module and a user module with the same residual take the SO3 route, with PCG() or sparse=True alone;
    # structured.recognize keeps returning None for SO3 graphs (the LM asks for the SO3 family where it would otherwise
    # build per-residual blocks)
    for m in (pp.module.PoseGraph(pp.SO3(cu(g["nodes0"]))), UserPoseGraph(pp.SO3(cu(g["nodes0"])))):
        assert type(rec(m, inp, list(m.parameters()), **kw)) is structured.SO3PGOProblem
        assert type(rec(m, inp, list(m.parameters()), solver=PCG())) is structured.SO3PGOProblem
        assert type(rec(m, inp, list(m.parameters()), sparse=True)) is structured.SO3PGOProblem
        assert structured.recognize(m, inp, list(m.parameters()), **kw) is None
        for lm_kw in (kw, dict(solver=PCG()), dict(sparse=True)):
            assert type(_problem_of(m, inp, **lm_kw)) is structured.SO3PGOProblem
    # information matrices, mixed dtypes, CPU tensors, GaussNewton: not the SO3 route
    m = pp.module.PoseGraph(pp.SO3(cu(g["nodes0"])))
    W = torch.eye(3, dtype=torch.float64, device="cuda").expand(len(e), 3, 3)
    assert rec(m, inp, list(m.parameters()), weight=W, **kw) is None
    assert not isinstance(_problem_of(m, inp, weight=W, **kw), structured.SO3PGOProblem)
    m = pp.module.PoseGraph(pp.SO3(cu(g["nodes0"])))
    assert rec(m, (e.cuda(), pp.SO3(cu(g["Z"], torch.float32))), list(m.parameters()), **kw) is None
    assert not isinstance(_problem_of(m, (e.cuda(), pp.SO3(cu(g["Z"], torch.float32))), **kw), structured.SO3PGOProblem)
    m = pp.module.PoseGraph(pp.SO3(torch.from_numpy(g["nodes0"])))
    cpu_inp = (e, pp.SO3(torch.from_numpy(g["Z"])))
    assert rec(m, cpu_inp, list(m.parameters()), **kw) is None
    assert not isinstance(_problem_of(m, cpu_inp, **kw), structured.SO3PGOProblem)
    m = pp.module.PoseGraph(pp.SO3(cu(g["nodes0"])))
    gn = pp.optim.GaussNewton(m)
    gn.step(input=inp)
    assert gn._problem is None
    # a process group, and no iterative solver asked for
    assert rec(m, inp, list(m.parameters()), group=True, **kw) is None
    assert rec(m, inp, list(m.parameters())) is None
    assert not isinstance(_problem_of(m, inp), structured.SO3PGOProblem)
    # RxSO3 graphs and so3 (algebra) parameters
    m = pp.module.PoseGraph(pp.randn_RxSO3(len(g["nodes0"]), dtype=torch.float64, device="cuda"))
    inp_r = (e.cuda(), pp.randn_RxSO3(len(e), dtype=torch.float64, device="cuda"))
    assert rec(m, inp_r, list(m.parameters()), **kw) is None
    assert not isinstance(_problem_of(m, inp_r, **kw), structured.SO3PGOProblem)
    m = UserPoseGraph(pp.randn_so3(len(g["nodes0"]), dtype=torch.float64, device="cuda"))
    assert rec(m, inp, list(m.parameters()), **kw) is None
    assert not isinstance(_problem_of(m, inp, **kw), structured.SO3PGOProblem)
    # a user module whose residual differs is not recognised
    class Other(UserPoseGraph):
        def forward(self, edges, poses):
            return 2.0 * super().forward(edges, poses)
    m = Other(pp.SO3(cu(g["nodes0"])))
    assert rec(m, inp, list(m.parameters()), **kw) is None
    assert not isinstance(_problem_of(m, inp, **kw), structured.SO3PGOProblem)
    # an out-of-range edge on the built-in module is an error, as on the other routes
    m = pp.module.PoseGraph(pp.SO3(cu(g["nodes0"])))
    bad = e.clone()
    bad[3, 1] = len(g["nodes0"])
    with pytest.raises(IndexError):
        rec(m, (bad.cuda(), inp[1]), list(m.parameters()), **kw)
    with pytest.raises(IndexError):
        pp.optim.LM(m, **kw).step(input=(bad.cuda(), inp[1]))
    # SE3 and Sim3 graphs keep their problem classes
    m = pp.module.PoseGraph(pp.randn_SE3(len(g["nodes0"]), dtype=torch.float64, device="cuda"))
    inp_t = (e.cuda(), pp.randn_SE3(len(e), dtype=torch.float64, device="cuda"))
    assert type(structured.recognize(m, inp_t, list(m.parameters()), **kw)) is structured.PGOProblem
    assert rec(m, inp_t, list(m.parameters()), **kw) is None
    m = pp.module.PoseGraph(pp.randn_Sim3(len(g["nodes0"]), dtype=torch.float64, device="cuda"))
    inp_s = (e.cuda(), pp.randn_Sim3(len(e), dtype=torch.float64, device="cuda"))
    assert type(structured.recognize(m, inp_s, list(m.parameters()), **kw)) is structured.Sim3PGOProblem
    assert rec(m, inp_s, list(m.parameters()), **kw) is None
