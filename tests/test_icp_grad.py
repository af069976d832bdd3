"""The ICP backward math (csrc/icp_math.cuh, host build) and its fp64 oracle (oracle/icp_grad_oracle.py) against the
reference's autograd (tests/golden/icp_grad.npz, oracle/make_golden_icp_grad.py) and torch fp64 autograd."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import icp_grad_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "icp_grad.npz"))
NAMES = sorted({k.split("/")[0] for k in GOLD.files})
_HOST = {}


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="icp_grad_host_")
        so = os.path.join(d, "icp_grad_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "icp_grad_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data)


def golden_case(name):
    p = f"{name}/"
    T = lambda k: torch.from_numpy(GOLD[p + k])   # noqa: E731
    o = int(GOLD[p + "ord"])
    init = T("init") if p + "init" in GOLD.files else None
    return T("source"), T("target"), init, math.inf if o == -1 else o, int(GOLD[p + "steps"]), T


def kabsch_adj(H, GR, eps=1e-12):
    H, GR = np.ascontiguousarray(H, np.float64), np.ascontiguousarray(GR, np.float64)
    out = np.zeros_like(H)
    _host().icp_host_kabsch_adj(_vp(H), ctypes.c_double(eps), _vp(GR), _vp(out), ctypes.c_longlong(H.shape[0]))
    return out


def kabsch(H, eps=1e-12):
    H = np.ascontiguousarray(H, np.float64)
    R = np.zeros(9)
    _host().icp_grad_host_kabsch(_vp(H), ctypes.c_double(eps), _vp(R))
    return R.reshape(3, 3)


def torch_kabsch_grad(H, GR, so3=False):
    """d <GR, R(H)> / dH by torch autograd: R = U Vh negated when det = -1 (svdtf), or (so3) U diag(1, 1, det U det V) Vh."""
    Ht = torch.tensor(H, dtype=torch.float64, requires_grad=True)
    U, S, Vh = torch.linalg.svd(Ht)
    if so3:
        d = torch.linalg.det(U).detach() * torch.linalg.det(Vh).detach()
        R = U @ torch.diag(torch.stack([torch.ones((), dtype=torch.float64), torch.ones((), dtype=torch.float64), d])) @ Vh
    else:
        R = U @ Vh
        if abs(float(torch.linalg.det(R)) + 1) < 1e-6:
            R = -R
    (R * torch.from_numpy(GR)).sum().backward()
    return Ht.grad.numpy()


def rand_rot(g):
    q = g.normal(size=4)
    return O.quat2mat(torch.from_numpy(q / np.linalg.norm(q))).numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the oracle is the reference's graph
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("loss", [0, 1])
def test_oracle_matches_reference_autograd(name, loss):
    src, tgt, init, o, K, T = golden_case(name)
    res, (gs, gt, gi) = O.grads(src, tgt, K, init, o, "reference", T("W"), T("probe"), T("w"), loss)
    np.testing.assert_allclose(res.numpy(), T("result").numpy(), rtol=0, atol=1e-13)
    for got, key in ((gs, f"gsrc{loss}"), (gt, f"gtgt{loss}")) + (((gi, f"ginit{loss}"),) if init is not None else ()):
        want = T(key).numpy()
        np.testing.assert_allclose(got.numpy(), want, rtol=0, atol=1e-12 * np.abs(want).max())


@pytest.mark.parametrize("name", NAMES)
def test_oracle_given_its_own_matches_is_bit_identical(name):
    """Replaying the matches the oracle found itself changes nothing: result and every gradient bit for bit."""
    src, tgt, init, o, K, T = golden_case(name)
    _, m = O.icp(src, tgt, K, init, o, "reference")
    assert len(m) == K
    for loss in (0, 1):
        a = O.grads(src, tgt, K, init, o, "reference", T("W"), T("probe"), T("w"), loss)
        b = O.grads(src, tgt, K, init, o, "reference", T("W"), T("probe"), T("w"), loss, matches=m)
        assert torch.equal(a[0], b[0])
        for x, y in zip(a[1], b[1]):
            assert (x is None and y is None) or torch.equal(x, y)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("loss", [0, 1])
def test_fixed_match_oracle_matches_reference_autograd(name, loss):
    """The fixed-match oracle, fed the matches of the reference's run, reproduces every golden."""
    src, tgt, init, o, K, T = golden_case(name)
    _, m = O.icp(src, tgt, K, init, o, "reference")
    res, (gs, gt, gi) = O.grads(src, tgt, K, init, o, "reference", T("W"), T("probe"), T("w"), loss, matches=m)
    np.testing.assert_allclose(res.numpy(), T("result").numpy(), rtol=0, atol=1e-13)
    for got, key in ((gs, f"gsrc{loss}"), (gt, f"gtgt{loss}")) + (((gi, f"ginit{loss}"),) if init is not None else ()):
        want = T(key).numpy()
        np.testing.assert_allclose(got.numpy(), want, rtol=0, atol=1e-12 * np.abs(want).max())


def test_fixed_match_oracle_follows_the_given_matches():
    """Matches other than the nearest ones change the result, and a wrong count of match tensors is refused."""
    src, tgt, init, o, K, T = golden_case(NAMES[0])
    res, m = O.icp(src, tgt, K, init, o)
    shifted = [torch.roll(x, 1, -1) for x in m]
    other, used = O.icp(src, tgt, K, init, o, matches=shifted)
    assert all(torch.equal(x, y) for x, y in zip(used, shifted))
    assert not torch.equal(res, other)
    with pytest.raises(ValueError):
        O.icp(src, tgt, K, init, o, matches=m[:-1])


@pytest.mark.parametrize("name", NAMES)
def test_goldens_use_the_agreeing_quaternion_branch(name):
    """In the goldens mat2SE3's quaternion has w >= 0, so the "project" rule of pp.module.ICP gives the same graph."""
    src, tgt, init, o, K, T = golden_case(name)
    for loss in (0, 1):
        a = O.grads(src, tgt, K, init, o, "reference", T("W"), T("probe"), T("w"), loss)[1]
        b = O.grads(src, tgt, K, init, o, "project", T("W"), T("probe"), T("w"), loss)[1]
        for x, y in zip(a, b):
            if x is not None:
                assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------------------------------
# host build of the adjoints against torch fp64 autograd
# ---------------------------------------------------------------------------------------------------------------------
def test_kabsch_adj_generic_and_negated():
    g = np.random.default_rng(1)
    seen = set()
    for _ in range(200):
        H = g.normal(size=(3, 3))
        GR = g.normal(size=(3, 3))
        want = torch_kabsch_grad(H, GR)
        got = kabsch_adj(H[None], GR[None])[0]
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-10 * max(1.0, np.abs(want).max()))
        seen.add(bool(np.linalg.det(H) < 0))
    assert seen == {True, False}                 # both the plain and the negated (det U V^T = -1) case


@pytest.mark.parametrize("sig", [(2.0, 2.0, 1.0), (3.0, 1.0, 1.0), (1.0, 1.0, 1.0), (2.0, 2.0, -1.0)])
def test_kabsch_adj_repeated_singular_values(sig):
    """Finite where torch's SVD backward is not: against central differences of the host Kabsch rule."""
    g = np.random.default_rng(2)
    for _ in range(5):
        H = rand_rot(g) @ np.diag(sig) @ rand_rot(g).T
        GR = g.normal(size=(3, 3))
        got = kabsch_adj(H[None], GR[None])[0]
        assert np.isfinite(got).all()
        h, num = 1e-6, np.zeros((3, 3))
        for a in range(3):
            for b in range(3):
                E = np.zeros((3, 3))
                E[a, b] = h
                num[a, b] = ((kabsch(H + E) - kabsch(H - E)) * GR).sum() / (2 * h)
        np.testing.assert_allclose(got, num, rtol=0, atol=1e-8 * max(1.0, np.abs(num).max()))


def test_kabsch_adj_planar_is_special_orthogonal_procrustes():
    """Rank 2: the derivative of U diag(1, 1, det U det V) V^T, whatever det U V^T the SVD would give."""
    g = np.random.default_rng(3)
    for k in range(100):
        sig = np.diag([2.0 + g.random(), 0.5 + g.random(), 0.0])
        H = rand_rot(g) @ sig @ rand_rot(g).T
        if k % 2:
            H = H @ np.diag([1.0, 1.0, -1.0])        # a reflection of the plane: same rank, other det sign of U V^T
        GR = g.normal(size=(3, 3))
        want = torch_kabsch_grad(H, GR, so3=True)
        got = kabsch_adj(H[None], GR[None])[0]
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-10 * max(1.0, np.abs(want).max()))


def test_kabsch_adj_collinear_and_zero_are_zero():
    g = np.random.default_rng(4)
    for _ in range(20):
        a, b = g.normal(size=3), g.normal(size=3)
        for H in (np.outer(a, b), np.zeros((3, 3))):
            assert np.array_equal(kabsch_adj(H[None], g.normal(size=(1, 3, 3)))[0], np.zeros((3, 3)))


def test_quat_ref_matches_oracle_every_branch_and_sign_rule():
    """mat2SE3's quaternion; where its w < 0, pp.module.ICP returns the negated quaternion (the w >= 0 rule)."""
    g = np.random.default_rng(5)
    Rs = np.stack([rand_rot(g) for _ in range(400)])
    q = np.zeros((len(Rs), 4))
    _host().icp_host_quat_ref(_vp(np.ascontiguousarray(Rs)), _vp(q), ctypes.c_longlong(len(Rs)))
    want = O.mat2quat_ref(torch.from_numpy(Rs)).numpy()
    np.testing.assert_allclose(q, want, rtol=0, atol=1e-14)
    assert (q[:, 3] < 0).any() and (q[:, 3] > 0).any()
    r = Rs
    branch = np.where(r[:, 2, 2] < 1e-5, np.where(r[:, 0, 0] > r[:, 1, 1], 0, 1), np.where(r[:, 0, 0] < -r[:, 1, 1], 2, 3))
    assert set(branch) == {0, 1, 2, 3}
    assert (q[branch == 3, 3] > 0).all()          # the trace branch always agrees with w >= 0


def _pts_sums(p, y, c0):
    d, e = p - c0, y - c0
    return np.concatenate([d.sum(0), e.sum(0), (e[:, :, None] * d[:, None, :]).sum(0).ravel(), [0.0, len(p)]])


@pytest.mark.parametrize("case", ["generic", "negated", "large_turn"])
def test_iter_adj_matches_torch_autograd(case):
    """One iteration's per-batch adjoint: the cotangents of the moved and matched points through svdtf, mat2SE3's
    quaternion and the Act convention [sum g, sum p x g, 0], against torch autograd of those formulas."""
    g = np.random.default_rng({"generic": 6, "negated": 7, "large_turn": 8}[case])
    n = 40
    p = g.normal(size=(n, 3)) + 3.0
    R0 = rand_rot(g) if case == "large_turn" else O.quat2mat(torch.tensor([0.05, -0.03, 0.02, 1.0]) / 1.0016).numpy()
    y = (p @ R0.T) + 0.3 + 0.05 * g.normal(size=(n, 3))
    if case == "negated":
        y = y * np.array([1.0, 1.0, -1.0])
    c0 = y[0].copy()
    gsum, om = g.normal(size=3), g.normal(size=3)
    P = np.zeros((3, 4))
    P[:, 3] = gsum
    P[2, 1], P[0, 2], P[1, 0] = om                 # sum p x g = (P21 - P12, P02 - P20, P10 - P01)
    out = np.zeros(30)
    _host().icp_host_iter_adj(_vp(_pts_sums(p, y, c0)), _vp(c0), ctypes.c_double(1e-12), _vp(np.ascontiguousarray(P)),
                              _vp(out), ctypes.c_longlong(1))
    pt, yt = torch.tensor(p, requires_grad=True), torch.tensor(y, requires_grad=True)
    T = O.svdtf(pt, yt)
    L = (T[:3] * torch.from_numpy(gsum)).sum() + (T[3:6] * torch.from_numpy(om)).sum()
    L.backward()
    GH, ms, mt, dms, dmt = out[9:18].reshape(3, 3), out[18:21], out[21:24], out[24:27], out[27:30]
    gp = (y - mt) @ GH + dms
    gy = (p - ms) @ GH.T + dmt
    np.testing.assert_allclose(gp, pt.grad.numpy(), rtol=0, atol=1e-10 * np.abs(pt.grad.numpy()).max())
    np.testing.assert_allclose(gy, yt.grad.numpy(), rtol=0, atol=1e-10 * np.abs(yt.grad.numpy()).max())


def test_final_adj_matches_torch_autograd():
    """The closing svdtf(source, p_K) with the quaternion pp.module.ICP returns (w >= 0), for a general [t, q] cotangent."""
    g = np.random.default_rng(9)
    for k in range(20):
        n = 30
        s = g.normal(size=(n, 3)) + 1.0
        R0 = rand_rot(g)
        e = s @ R0.T + g.normal(size=3) + 0.02 * g.normal(size=(n, 3))
        gout = g.normal(size=7)
        cs = s[0].copy()
        d, ee = s - cs, e - e[0]
        F = np.concatenate([d.sum(0), ee.sum(0), (ee[:, :, None] * d[:, None, :]).sum(0).ravel()])
        out = np.zeros(21)
        _host().icp_host_final_adj(_vp(F), _vp(cs), ctypes.c_double(n), ctypes.c_double(1e-12), _vp(gout), _vp(out),
                                   ctypes.c_longlong(1))
        st, et = torch.tensor(s, requires_grad=True), torch.tensor(e, requires_grad=True)
        (O.svdtf(st, et, "project") * torch.from_numpy(gout)).sum().backward()
        GH, md, me, dms, dmt = out[:9].reshape(3, 3), out[9:12], out[12:15], out[15:18], out[18:21]
        gs = (ee - me) @ GH + dms
        ge = (d - md) @ GH.T + dmt
        np.testing.assert_allclose(gs, st.grad.numpy(), rtol=0, atol=1e-10 * np.abs(st.grad.numpy()).max())
        np.testing.assert_allclose(ge, et.grad.numpy(), rtol=0, atol=1e-10 * np.abs(et.grad.numpy()).max())
