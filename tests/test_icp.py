"""pp.knn, pp.module.ICP and pp.utils.ReduceToBason (csrc/knn.cu, csrc/icp_math.cuh) against the reference goldens
(tests/golden/icp.npz, oracle/make_golden_icp.py) and the fp64 oracle (oracle/icp_oracle.py)."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import icp_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "icp.npz"))
ICP_NAMES = sorted({k.split("/")[1] for k in GOLD.files if k.startswith("icp/")})
KNN_NAMES = sorted({k.split("/")[1] for k in GOLD.files if k.startswith("knn/")})
STEP_NAMES = sorted({k.split("/")[1] for k in GOLD.files if k.startswith("stepper/")})
# In the L-wall scenes one batch element converges to an exact fit: its loss ends at ~1e-14 in fp64 (~1e-6 in fp32) and
# rounding noise decides the patience count from then on, so only the transform and the loss prefix are compared there.
NOISE_STOP = {"lwall_f32", "lwall_f64"}


def _ord(v):
    v = int(v)
    return math.inf if v == -1 else v


def _icp_case(name):
    p = f"icp/{name}/"
    init = GOLD[p + "init"] if p + "init" in GOLD.files else None
    return (GOLD[p + "source"], GOLD[p + "target"], init, int(GOLD[p + "ord"]), int(GOLD[p + "steps_max"]),
            int(GOLD[p + "patience"]))


def _mats(se3):
    return O.se3_to_mat(np.asarray(se3, np.float64)).reshape(-1, 3, 4)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: oracle vs goldens, stepper, host build of the Kabsch rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", KNN_NAMES)
def test_oracle_knn_matches_reference(name):
    p = f"knn/{name}/"
    v, i = O.knn(GOLD[p + "ref"], GOLD[p + "nbr"], int(GOLD[p + "k"]), _ord(GOLD[p + "ord"]), bool(GOLD[p + "largest"]))
    np.testing.assert_allclose(v, GOLD[p + "values"], rtol=1e-13, atol=1e-14)
    if not name.startswith("dups"):                 # with duplicates the reference's topk order among ties is its own
        np.testing.assert_array_equal(i, GOLD[p + "indices"])


@pytest.mark.parametrize("name", ICP_NAMES)
def test_oracle_icp_matches_reference(name):
    src, tgt, init, ordv, steps, patience = _icp_case(name)
    f32 = name.endswith("f32")
    A, L, _ = O.icp(src, tgt, None if init is None else _mats(init), ordv, steps, patience,
                    eps=O.KABSCH_EPS[np.float32 if f32 else np.float64])
    ref_losses = GOLD[f"icp/{name}/losses"].reshape(len(GOLD[f"icp/{name}/losses"]), -1)
    n = min(len(L), len(ref_losses))
    tol = 2e-5 if f32 else 1e-12
    np.testing.assert_allclose(L[:n].reshape(n, -1), ref_losses[:n], rtol=tol, atol=tol)
    np.testing.assert_allclose(A, _mats(GOLD[f"icp/{name}/result"]), atol=2e-5 if f32 else 1e-12)
    if name not in NOISE_STOP:
        assert len(L) == int(GOLD[f"icp/{name}/steps"])


@pytest.mark.parametrize("name", STEP_NAMES)
def test_reduce_to_bason_reproduces_reference_traces(name):
    steps, patience, dec, tol = GOLD[f"stepper/{name}/kw"]
    losses, trace = GOLD[f"stepper/{name}/losses"], GOLD[f"stepper/{name}/trace"]
    st = pp.utils.ReduceToBason(int(steps), patience=int(patience), decreasing=float(dec), tol=float(tol))
    got = []
    for l in losses:
        if not st.continual():
            break
        st.step(torch.tensor(l))
        got.append((st.steps, st.patience_count, int(st.continual())))
    np.testing.assert_array_equal(np.array(got), trace)
    # the device rule, host-compiled from icp_math.cuh, takes the same decisions
    is64 = losses.dtype == np.float64
    last = np.full(np.atleast_1d(losses[0]).shape, np.inf, dtype=losses.dtype)
    s = np.array([0.0, 0.0, 1.0])
    got = []
    for l in losses:
        if s[2] == 0.0:
            break
        l = np.ascontiguousarray(np.atleast_1d(l))
        _host().icp_host_r2b(int(is64), _vp(l), _vp(last), ctypes.c_longlong(l.size), _vp(s), ctypes.c_longlong(int(steps)),
                             ctypes.c_longlong(int(patience)), ctypes.c_double(dec), ctypes.c_double(tol))
        got.append((int(s[0]), int(s[1]), int(s[2])))
    np.testing.assert_array_equal(np.array(got), trace)


_HOST = {}


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data)


def _host():
    if "lib" not in _HOST:
        import tempfile
        d = tempfile.mkdtemp(prefix="icp_host_")
        so = os.path.join(d, "libicphost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "icp_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def host_kabsch(H, eps):
    H = np.ascontiguousarray(H, np.float64).reshape(-1, 9)
    R = np.empty_like(H)
    _host().icp_host_kabsch(_vp(H), ctypes.c_double(eps), _vp(R), ctypes.c_longlong(H.shape[0]))
    return R.reshape(-1, 3, 3)


def _rot(rng):
    q = rng.standard_normal(4)
    return O.quat2mat(q / np.linalg.norm(q))


def _scenes(rng):
    """(name, source (N,3), target (N,3)) for each rank class."""
    out = []
    R, t = _rot(rng), rng.standard_normal(3)
    s = rng.standard_normal((50, 3))
    out.append(("rank3", s, s @ R.T + t + 0.01 * rng.standard_normal((50, 3))))
    out.append(("reflection", s, s * np.array([1.0, 1.0, -1.0]) @ R.T))
    p = np.c_[rng.standard_normal((40, 2)), np.zeros(40)]
    out.append(("planar", p, p @ R.T + t))
    out.append(("planar_reflected", p, (p * np.array([1.0, -1.0, 0.0])) @ R.T))
    line = np.outer(np.linspace(-1, 2, 7), rng.standard_normal(3))
    out.append(("collinear", line, line @ R.T + t))
    out.append(("collinear_reversed", line, -line + t))
    out.append(("docstring", np.array([[0.0, 0, 0], [1, 0, 0], [2, 0, 0]]),
                np.array([[0.2, 0.1, 0.0], [1.1397, 0.442, 0.0], [2.0794, 0.7840, 0.0]])))
    c = np.tile(rng.standard_normal(3), (5, 1))
    out.append(("coincident", c, c + 1.0))
    return out


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kabsch_rule_host_build(seed):
    rng = np.random.default_rng(seed)
    for name, s, t in _scenes(rng):
        cs, ct = s - s.mean(0), t - t.mean(0)
        H = ct.T @ cs
        R = host_kabsch(H, 1e-12)[0]
        np.testing.assert_allclose(R, O.kabsch(H, 1e-12), atol=1e-9, err_msg=name)
        np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-12, err_msg=name)
        sv = np.linalg.svd(H, compute_uv=False)
        if name in ("rank3", "reflection"):         # unique optimum of the reference rule: U V^T (negated if improper)
            U, _, Vt = np.linalg.svd(H)
            Rr = U @ Vt
            Rr = -Rr if abs(np.linalg.det(Rr) + 1) < 1e-6 else Rr
            np.testing.assert_allclose(O.kabsch_cost(R, s, t), O.kabsch_cost(Rr, s, t), rtol=1e-10, atol=1e-10)
        else:                                      # rank-deficient: a proper rotation with the optimal cost
            assert abs(np.linalg.det(R) - 1.0) < 1e-10, name
            best = ((ct ** 2).sum() + (cs ** 2).sum()) - 2 * sv.sum()
            assert O.kabsch_cost(R, s, t) <= best + 1e-9 * (1 + abs(best)), name
    # the docstring example (collinear source): a rotation about z, 20 degrees
    _, s, t = _scenes(np.random.default_rng(0))[6]
    R = host_kabsch((t - t.mean(0)).T @ (s - s.mean(0)), 1e-6)[0]
    np.testing.assert_allclose(R[2], [0, 0, 1], atol=1e-4)
    assert abs(math.degrees(math.atan2(R[1, 0], R[0, 0])) - 20.0) < 0.1
    assert (host_kabsch(np.zeros((3, 3)), 1e-12)[0] == np.eye(3)).all()


def test_knn_and_icp_reject_bad_arguments_on_cpu():
    a = torch.randn(5, 3)
    with pytest.raises(NotImplementedError, match="CPU"):
        pp.knn(a, a)
    with pytest.raises(NotImplementedError, match="CPU"):
        pp.module.ICP()(a, a)


def test_icp_init_on_another_device_is_copied_before_the_launch():
    """An init on another device than the clouds (a CPU pp.identity_SE3(B), say) reaches the kernels as rows on the
    clouds' device; a non-SE3 init is refused."""
    from pypose_b200.module.icp import _init_rows
    init = pp.SE3(torch.tensor([[0.1, 0.2, 0.3, 0.0, 0.0, 0.0, 1.0], [0.0, 0.0, 0.0, 0.0, 0.6, 0.0, 0.8]]))
    rows = _init_rows(init, torch.Size([2]), torch.device("meta"), torch.float32)
    assert rows.device.type == "meta" and rows.dtype == torch.float32 and rows.shape == (2, 7)
    rows = _init_rows(init[:1], torch.Size([3]), torch.device("cpu"), torch.float64)
    assert rows.shape == (1, 7) and rows.dtype == torch.float64
    with pytest.raises(TypeError):
        pp.module.ICP(init=pp.so3(torch.zeros(1, 3)))
    with pytest.raises(TypeError):
        pp.module.ICP(init=torch.zeros(1, 7))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: knn
# ---------------------------------------------------------------------------------------------------------------------
def _check_knn(r, n, k, ordv, largest, dt):
    got = pp.knn(r, n, k=k, ord=ordv, largest=largest)
    v, i = got.values.cpu().numpy(), got.indices.cpu().numpy()
    rv, ri = O.knn(r.double().cpu().numpy(), n.double().cpu().numpy(), k, ordv, largest)
    assert got.indices.dtype == torch.int64 and v.shape == rv.shape
    if dt == torch.float64:
        np.testing.assert_array_equal(i, ri)
        np.testing.assert_allclose(v, rv, rtol=1e-13, atol=1e-14)
    else:
        np.testing.assert_allclose(v, rv, rtol=1e-6, atol=1e-6)
        # indices may differ only where neighbouring fp64 distances are within fp32 rounding
        d = O.distances(r.double().cpu().numpy(), n.double().cpu().numpy(), ordv)
        dg = np.take_along_axis(d, i, -1)
        np.testing.assert_allclose(dg, rv, rtol=2e-6, atol=2e-6)
        full = np.sort(-d if largest else d, -1)
        pad = np.full(full.shape[:-1] + (1,), np.inf)
        ext = np.concatenate([-pad, full, pad], -1)
        thr = 1e-5 * (1 + np.abs(full[..., :k]))
        clear = (ext[..., 1:k + 1] - ext[..., :k] > thr) & (ext[..., 2:k + 2] - ext[..., 1:k + 1] > thr)
        assert (i[clear] == ri[clear]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [2, 3, 5])
@pytest.mark.parametrize("ordv", [1, 2, math.inf])
def test_knn_vs_oracle(dt, D, ordv):
    g = torch.Generator().manual_seed(D * 10 + (3 if ordv == math.inf else ordv))
    dev = "cuda"
    for (B, N1, N2) in ((2, 300, 333), (1, 257, 1), (3, 1, 70)):
        r = torch.randn(B, N1, D, generator=g, dtype=torch.float64).to(dt).to(dev)
        n = torch.randn(B, N2, D, generator=g, dtype=torch.float64).to(dt).to(dev)
        for k in sorted({1, 4, 32, N2}):
            if k > N2 or k > 32:
                continue
            for largest in (False, True):
                _check_knn(r, n, k, ordv, largest, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_knn_goldens_broadcast_noncontiguous_and_empty(dt):
    for name in KNN_NAMES:
        p = f"knn/{name}/"
        r = torch.from_numpy(GOLD[p + "ref"]).to(dt).cuda()
        n = torch.from_numpy(GOLD[p + "nbr"]).to(dt).cuda()
        k, ordv, largest = int(GOLD[p + "k"]), _ord(GOLD[p + "ord"]), bool(GOLD[p + "largest"])
        got = pp.knn(r, n, k=k, ord=ordv, largest=largest)
        np.testing.assert_allclose(got.values.cpu().double().numpy(), GOLD[p + "values"],
                                   rtol=1e-6 if dt == torch.float32 else 1e-13, atol=1e-6 if dt == torch.float32 else 1e-14)
        if dt == torch.float64:                      # duplicates: lower index first
            _, ri = O.knn(r.cpu().numpy(), n.cpu().numpy(), k, ordv, largest)
            np.testing.assert_array_equal(got.indices.cpu().numpy(), ri)
    # broadcast batches both ways, non-contiguous inputs
    g = torch.Generator().manual_seed(3)
    base = torch.randn(4, 3, 90, 6, generator=g, dtype=torch.float64).to(dt).cuda()
    r = base[:, :1, :, 1:4]                          # (4, 1, 90, 3), strided
    n = torch.randn(5, 1, 120, 3, generator=g, dtype=torch.float64).to(dt).cuda().transpose(0, 1)   # (1, 5, 120, 3)
    got = pp.knn(r, n, k=7)
    assert got.values.shape == (4, 5, 90, 7)
    _check_knn(r.expand(4, 5, 90, 3).reshape(20, 90, 3), n.expand(4, 5, 120, 3).reshape(20, 120, 3), 7, 2, False, dt)
    rv, ri = O.knn(r.double().cpu().numpy(), n.double().cpu().numpy(), 7, 2)
    np.testing.assert_allclose(got.values.cpu().double().numpy(), rv, rtol=1e-6, atol=1e-6)
    # empty batch / no queries
    e = pp.knn(torch.empty(0, 10, 3, dtype=dt, device="cuda"), torch.randn(1, 10, 3, dtype=dt, device="cuda"), k=2)
    assert e.values.shape == (0, 10, 2) and e.indices.shape == (0, 10, 2)
    e = pp.knn(torch.empty(2, 0, 3, dtype=dt, device="cuda"), torch.randn(2, 10, 3, dtype=dt, device="cuda"), k=2)
    assert e.values.shape == (2, 0, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_knn_split_path_large_and_bit_reproducible(dt):
    g = torch.Generator().manual_seed(17)
    r = torch.rand(1, 20000, 3, generator=g, dtype=torch.float64).to(dt).cuda()
    n = torch.rand(1, 200000, 3, generator=g, dtype=torch.float64).to(dt).cuda()
    for k in (1, 8):
        a = pp.knn(r, n, k=k)
        b = pp.knn(r, n, k=k)
        assert torch.equal(a.values, b.values) and torch.equal(a.indices, b.indices)
        sub = torch.arange(0, 20000, 97)
        _check_knn(r[:, sub], n, k, 2, False, dt)
        np.testing.assert_array_equal(a.indices[:, sub].cpu().numpy(), pp.knn(r[:, sub], n, k=k).indices.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_knn_split_path_merge_every_mode(dt):
    """The merge kernel with -inf initial lists (largest), unsquared values (ord 1 / inf) and K = 32: few queries against
    many targets so that the N2 range is split; a subsample of the queries is compared with the oracle."""
    g = torch.Generator().manual_seed(23)
    r = torch.rand(2, 3000, 3, generator=g, dtype=torch.float64).to(dt).cuda()
    n = torch.rand(2, 60000, 3, generator=g, dtype=torch.float64).to(dt).cuda()
    q = _C_knn_ws(2, 3000, 60000, 3, 32, r.element_size())
    assert q > 0                                     # the split path is taken
    sub = torch.arange(0, 3000, 61)
    for k, ordv, largest in ((32, math.inf, True), (4, 1, False), (32, 2, True), (17, 1, True)):
        a = pp.knn(r, n, k=k, ord=ordv, largest=largest)
        b = pp.knn(r, n, k=k, ord=ordv, largest=largest)
        assert torch.equal(a.values, b.values) and torch.equal(a.indices, b.indices)
        rs = r[:, sub].double().cpu().numpy()
        rv, ri = O.knn(rs, n.double().cpu().numpy(), k, ordv, largest)
        v, i = a.values[:, sub].double().cpu().numpy(), a.indices[:, sub].cpu().numpy()
        if dt == torch.float64:
            np.testing.assert_array_equal(i, ri)
            np.testing.assert_allclose(v, rv, rtol=1e-13, atol=1e-14)
        else:
            np.testing.assert_allclose(v, rv, rtol=1e-6, atol=1e-6)
            dg = np.take_along_axis(O.distances(rs, n.double().cpu().numpy(), ordv), i, -1)
            np.testing.assert_allclose(dg, rv, rtol=2e-6, atol=2e-6)


def _C_knn_ws(B, N1, N2, D, k, elem):
    import ctypes as ct
    from pypose_b200 import _C
    f = _C.lib().b200_knn_workspace_bytes
    f.restype, f.argtypes = ct.c_longlong, [ct.c_longlong] * 6
    with torch.cuda.device(0):
        return int(f(B, N1, N2, D, k, elem))


@pytest.mark.gpu
def test_knn_nan_query_leaves_empty_slots_and_gradient_is_safe():
    r = torch.randn(1, 6, 3, dtype=torch.float64, device="cuda")
    r[0, 2, 1] = float("nan")
    n = torch.randn(1, 9, 3, dtype=torch.float64, device="cuda", requires_grad=True)
    out = pp.knn(r, n, k=2)
    assert (out.indices[0, 2] == -1).all() and torch.isinf(out.values[0, 2]).all()
    assert (out.indices[0, [0, 1, 3, 4, 5]] >= 0).all()
    out.values[torch.isfinite(out.values)].sum().backward()
    torch.cuda.synchronize()
    assert torch.isfinite(n.grad).all()


@pytest.mark.gpu
def test_knn_values_gradient_and_errors():
    g = torch.Generator().manual_seed(2)
    r = torch.randn(2, 40, 3, generator=g, dtype=torch.float64).cuda().requires_grad_()
    n = torch.randn(2, 50, 3, generator=g, dtype=torch.float64).cuda().requires_grad_()
    for ordv in (1, 2, math.inf):
        out = pp.knn(r, n, k=3, ord=ordv)
        w = torch.randn_like(out.values)
        gr, gn = torch.autograd.grad((out.values * w).sum(), (r, n))
        d = torch.linalg.vector_norm(r.unsqueeze(-2) - n.unsqueeze(-3), ord=ordv, dim=-1)
        ref = torch.gather(d, -1, out.indices)
        er, en = torch.autograd.grad((ref * w).sum(), (r, n))
        torch.testing.assert_close(gr, er, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(gn, en, rtol=1e-12, atol=1e-12)
    a = torch.randn(3, 4, 3, device="cuda")
    for kw, exc in ((dict(dim=0), ValueError), (dict(ord=3), ValueError), (dict(k=33), ValueError), (dict(k=5), ValueError)):
        with pytest.raises(exc):
            pp.knn(a, a, **kw)
    with pytest.raises(ValueError):
        pp.knn(a, a.double())
    with pytest.raises(NotImplementedError):
        pp.knn(a, a.cpu())


# ---------------------------------------------------------------------------------------------------------------------
# GPU: ICP
# ---------------------------------------------------------------------------------------------------------------------
def _run_icp(name, stepper_cls=pp.utils.ReduceToBason, **skw):
    src, tgt, init, ordv, steps, patience = _icp_case(name)
    st = stepper_cls(steps, patience=patience, **skw)
    icp = pp.module.ICP(stepper=st)
    i = None if init is None else pp.SE3(torch.from_numpy(init).cuda())
    out = icp(torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(), ord=ordv, init=i)
    return out, st


class _Recording(pp.utils.ReduceToBason):
    """Not exactly ReduceToBason: ICP takes the host loop and calls step() every iteration."""

    def reset(self):
        super().reset()
        self.losses = []

    def step(self, loss):
        self.losses.append(loss.detach().cpu().numpy().copy())
        super().step(loss)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ICP_NAMES)
def test_icp_vs_reference_goldens(name):
    f32 = name.endswith("f32")
    out, st = _run_icp(name, _Recording)
    got = _mats(out.tensor().cpu().numpy())
    np.testing.assert_allclose(got, _mats(GOLD[f"icp/{name}/result"]), atol=2e-5 if f32 else 1e-9)
    ref_losses = GOLD[f"icp/{name}/losses"].reshape(len(GOLD[f"icp/{name}/losses"]), -1)
    n = min(len(st.losses), len(ref_losses))
    np.testing.assert_allclose(np.array(st.losses[:n]).reshape(n, -1), ref_losses[:n], rtol=2e-5 if f32 else 1e-9,
                               atol=2e-5 if f32 else 1e-12)
    if name not in NOISE_STOP and not f32:
        assert st.steps == int(GOLD[f"icp/{name}/steps"])
    # the device-decided loop: same steps, bit-identical transform, same stepper state as the host loop
    out2, st2 = _run_icp(name)
    assert st2.steps == st.steps and st2.patience_count == st.patience_count and st2.continual() == st.continual()
    assert torch.equal(out2.tensor(), out.tensor())
    assert torch.equal(st2.last.reshape(-1), st.last.reshape(-1))


@pytest.mark.gpu
def test_icp_cpu_init_with_cuda_clouds():
    src, tgt, init, ordv, steps, patience = _icp_case("init_f64")
    res = []
    for dev in ("cpu", "cuda"):
        st = pp.utils.ReduceToBason(steps, patience=patience)
        out = pp.module.ICP(init=pp.SE3(torch.from_numpy(init).to(dev)), stepper=st)(
            torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(), ord=ordv)
        res.append(out.tensor())
    assert torch.equal(res[0], res[1])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_icp_large_converges_and_final_matches_agree_with_oracle(dt):
    g = torch.Generator().manual_seed(21)
    N = 100000
    xy = torch.rand(N, 2, generator=g, dtype=torch.float64) * 10           # a curved surface: z = sin x + cos 0.7 y
    tgt = torch.cat([xy, (torch.sin(xy[:, :1]) + torch.cos(0.7 * xy[:, 1:]))], 1)[None].to(dt)
    tf = pp.se3(torch.tensor([[0.2, -0.1, 0.05, 0.01, -0.01, 0.02]], dtype=torch.float64, device="cuda")).Exp()
    src = tf.Inv().unsqueeze(-2).Act(tgt.double().cuda()).to(dt).cpu()   # tgt = tf src exactly (up to rounding)
    st = pp.utils.ReduceToBason(100)
    out = pp.module.ICP(stepper=st)(src.cuda(), tgt.cuda())
    A = _mats(out.tensor().double().cpu().numpy())[0]
    T = _mats(tf.tensor().cpu().numpy())[0]
    np.testing.assert_allclose(A, T, atol=1e-4 if dt == torch.float32 else 1e-8)
    # The match kernel's own correspondences are not exposed.  What is checked: with the returned A applied on the host in
    # fp64, pp.knn matches a 1e3-query subsample as the fp64 oracle does (wherever the nearest target is unambiguous).
    sub = torch.arange(0, N, N // 1000)
    P = src[0, sub].double().numpy() @ A[:, :3].T + A[:, 3]
    Pd = torch.from_numpy(P).to(dt)
    got = pp.knn(Pd.cuda(), tgt[0].cuda()).indices[:, 0].cpu().numpy()
    d = O.distances(Pd.double().numpy(), tgt[0].double().numpy())
    _, ri = O.knn(Pd.double().numpy(), tgt[0].double().numpy(), 1)
    srt = np.sort(d, -1)
    clear = (srt[:, 1] - srt[:, 0]) > 1e-5
    assert clear.mean() > 0.9 and (got[clear] == ri[clear, 0]).all()
