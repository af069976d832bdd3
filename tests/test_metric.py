"""pp.metric.ape / rpe (csrc/traj.cu, csrc/traj_math.cuh) against reference goldens (oracle/make_golden_metric.py) and the
numpy oracle (oracle/metric_oracle.py).  DESIGN.md §3.6."""
import ctypes
import json
import math
import os
import subprocess
import tempfile
import warnings

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from pypose_b200.metric import ape_rpe as A
from oracle import metric_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "metric.npz"))
CASES = json.loads(str(GOLD["cases"]))
NAMES = list(CASES)
REF_NAMES = [n for n in NAMES if CASES[n]["from"] == "reference"]
_HOST = {}


def case(name):
    """fn, rstamp, rpose, estamp, epose, kwargs of a golden case; inputs are rebuilt from their recipes"""
    c = CASES[name]
    get = lambda k: O.synth(c[k], GOLD) if k in c else None   # noqa: E731
    return c["fn"], get("rstamp"), get("rpose"), get("estamp"), get("epose"), c["kw"]


def gidx(name, k):
    """the reference's association (m1 short, m2 long) or pair (src, tgt) indices of a golden case"""
    return np.cumsum(GOLD[CASES[name][k]], dtype=np.int64)


def oracle_kw(kw):
    """keyword arguments of pp.metric -> those of the oracle"""
    m = {"align": "align_", "associate": "associate_"}
    return {m.get(k, k): v for k, v in kw.items() if k not in ("otype", "thresh")}


def gold_stats(name, otype):
    s = CASES[name]["stats"]
    return dict(zip(O.KEYS, s)) if otype == 'All' else {otype: s[0]}


def close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.all((np.abs(a - b) <= tol * (1 + np.abs(b))) | (np.isnan(a) & np.isnan(b)))


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="metric_host_")
        so = os.path.join(d, "libmetrichost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "metric_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def host_path(t):
    t = np.ascontiguousarray(t, np.float64)
    n = len(t)
    l, D = np.empty(max(n - 1, 0)), np.empty(n)
    _host().metric_host_path(_vp(t), ctypes.c_longlong(n), _vp(l), _vp(D))
    return l, D


def host_match(short, long_, off, diff):
    short, long_ = np.ascontiguousarray(short, np.float64), np.ascontiguousarray(long_, np.float64)
    j, keep = np.empty(len(short), np.int64), np.empty(len(short), np.uint8)
    _host().metric_host_match(_vp(short), ctypes.c_longlong(len(short)), _vp(long_), ctypes.c_longlong(len(long_)),
                              ctypes.c_double(off), ctypes.c_double(diff), _vp(j), _vp(keep))
    return j, keep.astype(bool)


def host_pairs(D, delta, tol):
    n = len(D)
    j, keep = np.empty(max(n - 1, 0), np.int64), np.empty(max(n - 1, 0), np.uint8)
    _host().metric_host_pairs(_vp(D), ctypes.c_longlong(n), ctypes.c_double(delta), ctypes.c_double(tol), _vp(j), _vp(keep))
    keep = keep.astype(bool)
    return np.nonzero(keep)[0], j[keep]


def host_err(r, rb, e, eb, S, etype):
    c = lambda a: None if a is None else np.ascontiguousarray(a, np.float64)   # noqa: E731
    r, rb, e, eb, S = c(r), c(rb), c(e), c(eb), c(S)
    out = np.empty(len(r))
    _host().metric_host_err(_vp(r), _vp(rb), _vp(e), _vp(eb), _vp(S), ctypes.c_longlong(len(r)),
                            ctypes.c_int(O.ETYPES.index(etype)), _vp(out))
    return out


def stamps_of(rs, es, n_r, n_e):
    return (np.arange(n_r, dtype=np.float64) if rs is None else rs.astype(np.float64),
            np.arange(n_e, dtype=np.float64) if es is None else es.astype(np.float64))


# ------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", REF_NAMES)
def test_oracle_reproduces_reference_goldens(name):
    fn, rs, rp, es, ep, kw = case(name)
    rs, es = stamps_of(rs, es, len(rp), len(ep))
    r_idx, e_idx, _ = O.associate(rs, es, kw.get("diff", 0.01), kw.get("offset", 0.0))
    snd_longer = len(es) > len(rs)
    m1, m2 = gidx(name, "m1"), gidx(name, "m2")
    np.testing.assert_array_equal((r_idx, e_idx), (m1, m2) if snd_longer else (m2, m1))
    okw = oracle_kw(kw)
    if fn == "ape":
        err, *_ = O.ape(rs, rp, es, ep, **okw)
    else:
        err, src, tgt = O.rpe(rs, rp, es, ep, **okw)
        np.testing.assert_array_equal(src, gidx(name, "src"))
        np.testing.assert_array_equal(tgt, gidx(name, "tgt"))
    if "err" in CASES[name]:                   # stored up to 400 pairs; longer ones are pinned by the statistics
        assert close(err, GOLD[CASES[name]["err"]])
    st = O.stats(err)
    for k, v in gold_stats(name, kw.get("otype", "All")).items():
        assert close(st[k], v), (k, st[k], v)


def test_docstring_example_values():
    assert CASES["doc_ape"]["stats"][0] == 2.059025356439517
    assert CASES["doc_rpe"]["stats"][1] == CASES["doc_rpe"]["stats"][3] == 0.002306314257097237
    np.testing.assert_array_equal(gidx("doc_ape", "m2"), [0, 0, 0])        # every fp32 stamp ties: long index 0


@pytest.mark.parametrize("name", REF_NAMES)
def test_host_association_matches_reference(name):
    fn, rs, rp, es, ep, kw = case(name)
    rs, es = stamps_of(rs, es, len(rp), len(ep))
    snd_longer = len(es) > len(rs)
    short, long_ = (rs, es) if snd_longer else (es, rs)
    off = kw.get("offset", 0.0) if snd_longer else -kw.get("offset", 0.0)
    j, keep = host_match(short, long_, off, kw.get("diff", 0.01))
    np.testing.assert_array_equal(np.nonzero(keep)[0], gidx(name, "m1"))
    np.testing.assert_array_equal(j[keep], gidx(name, "m2"))


def test_host_path_lengths_are_the_references_bit_for_bit():
    g = torch.Generator().manual_seed(1)
    for n in (2, 3, 1000, 20000):
        t = torch.randn(n, 3, generator=g, dtype=torch.float64) * torch.tensor([1.0, 1e-3, 1e3], dtype=torch.float64)
        t[n // 3: n // 2] = t[n // 3]                       # a stationary run
        l, D = host_path(t.numpy())
        ref_l = torch.linalg.norm(t[:-1] - t[1:], dim=-1, dtype=torch.float64)      # the reference's formulation
        ref_D = torch.cat((torch.zeros(1, dtype=torch.float64), torch.cumsum(ref_l, dim=0)))
        np.testing.assert_array_equal(l, ref_l.numpy())
        np.testing.assert_array_equal(D, ref_D.numpy())
        np.testing.assert_array_equal(D, O.accumulated(t.numpy()))


@pytest.mark.parametrize("name", [n for n in REF_NAMES if "dist_all1_rpair1" in n or n == "large_rpe_dist"])
def test_host_distance_pairs_match_reference(name):
    fn, rs, rp, es, ep, kw = case(name)
    rs, es = stamps_of(rs, es, len(rp), len(ep))
    r_idx, _, _ = O.associate(rs, es)
    _, D = host_path(rp[r_idx, :3])
    src, tgt = host_pairs(D, kw["delta"], kw["delta"] * kw.get("rtol", 0.1))
    np.testing.assert_array_equal(src, gidx(name, "src"))
    np.testing.assert_array_equal(tgt, gidx(name, "tgt"))


@pytest.mark.parametrize("etype", O.ETYPES)
def test_host_errors_match_oracle(etype):
    g = np.random.default_rng(3)
    n = 500
    q = g.normal(size=(4, n, 4))
    q[..., 3] += 2.0
    q /= np.linalg.norm(q, axis=-1, keepdims=True)
    q[:2] = q[:2].astype(np.float32)                     # non-unit to fp64 precision
    P = np.concatenate([g.normal(size=(4, n, 3)), q], -1)
    P[3, :5, 3:] = [0.0, 0.0, 0.0, 1.0]                  # identity rotations
    P[3, 5:10, 3:] = [0.0, 1.0, 0.0, 0.0]                # half turns: the other mat2SO3 branches
    S = np.array([0.3, -0.2, 1.0, 0.1, -0.2, 0.3, 0.9273618495495703, 1.3])
    S[3:7] /= np.linalg.norm(S[3:7])
    for s in (None, S):
        assert close(host_err(P[0], None, P[1], None, s, etype), O.ape_errors(P[0], O.align(s, P[1]), etype))
        assert close(host_err(P[0], P[2], P[1], P[3], s, etype),
                     O.rpe_errors(P[0], P[2], O.align(s, P[1]), O.align(s, P[3]), etype))


def test_frame_pairs_never_reach_a_kernel():
    for n in (1, 2, 3, 10, 11):
        for d in (1, 3):
            for a in (False, True):
                src, tgt = A._pairs_by_frames(n, d, a, torch.device("cpu"))
                osrc, otgt = O.pairs_by_frames(n, d, a)
                np.testing.assert_array_equal(src.numpy(), osrc)
                np.testing.assert_array_equal(tgt.numpy(), otgt)
    with pytest.raises(ValueError):
        A._pairs_by_frames(10, 0.5, False, torch.device("cpu"))


def test_argument_validation():
    P = pp.identity_SE3(4)
    with pytest.raises(NotImplementedError):
        pp.metric.ape(None, P, None, P)                  # no CPU path
    with pytest.raises(ValueError):
        pp.metric.ape(None, P, None, P, etype="bogus")
    with pytest.raises(ValueError):
        pp.metric.rpe(None, P, None, P, otype="median")
    with pytest.raises(ValueError):
        pp.metric.rpe(None, P, None, P, associate="time")
    with pytest.raises(ValueError):
        pp.metric.ape(None, pp.identity_SO3(4), None, P)
    with pytest.raises(ValueError):
        pp.metric.ape(None, pp.identity_SE3(2, 4), None, P)


# ------------------------------------------------------------------------------------------------------------- GPU
DEV = torch.device("cuda:0")


def run_metric(fn, rs, rp, es, ep, kw, dtype=None):
    t = lambda a: None if a is None else torch.from_numpy(np.asarray(a)).to(DEV)   # noqa: E731
    P = lambda a: pp.SE3(t(a) if dtype is None else t(a).to(dtype))             # noqa: E731
    return getattr(pp.metric, fn)(t(rs), P(rp), t(es), P(ep), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_golden_cases_end_to_end(name):
    fn, rs, rp, es, ep, kw = case(name)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = run_metric(fn, rs, rp, es, ep, kw)
    if "warned" in CASES[name]:
        assert CASES[name]["warned"] == any("not enough" in str(x.message) for x in w)
    otype = kw.get("otype", "All")
    got = out if otype == "All" else {otype: out}
    if otype == "All":
        assert list(got) == O.KEYS
    for k, v in gold_stats(name, otype).items():
        assert got[k].dtype == torch.float64 and got[k].dim() == 0 and got[k].device == DEV
        assert close(got[k].item(), v, 1e-10 if kw.get("align") or kw.get("scale") else 1e-12), (k, got[k].item(), v)


def _kernel_assoc(rs, es, diff, offset):
    """(r_idx, e_idx) from b200_traj_match with the reference's short/long rule, empty when nothing matches"""
    rs, es = torch.from_numpy(rs).to(DEV), torch.from_numpy(es).to(DEV)
    snd_longer = len(es) > len(rs)
    short, long_ = (rs, es) if snd_longer else (es, rs)
    ns = len(short)
    ws = A._ws(ns, DEV)
    i_s, i_l, info = (torch.empty(k, dtype=torch.long, device=DEV) for k in (ns, ns, 3))
    pp._C.check(pp._C.fn("b200_traj_match")(short.data_ptr(), ns, long_.data_ptr(), len(long_),
                                            offset if snd_longer else -offset, diff, ws.data_ptr(), i_s.data_ptr(),
                                            i_l.data_ptr(), info.data_ptr(), pp._C.stream_ptr(DEV)), "match")
    cnt, bad_s, bad_l = info.tolist()
    assert not bad_s and not bad_l
    i_s, i_l = i_s[:cnt].cpu().numpy(), i_l[:cnt].cpu().numpy()
    return (i_s, i_l) if snd_longer else (i_l, i_s)


@pytest.mark.gpu
@pytest.mark.parametrize("ns,nl", [(1, 1), (5, 3), (1000, 1000), (10**6, 3 * 10**6)])
def test_association_equals_oracle(ns, nl):
    g = np.random.default_rng(ns)
    long_ = np.sort(np.round(g.uniform(0, nl / 100, nl), 3))          # a 1 ms grid: many duplicates
    short = np.sort(np.round(g.uniform(-1, nl / 100 + 1, ns) * 4) / 4)  # quarter steps: distances equal to diff = 0.25
    short[: ns // 3] = np.sort(g.choice(long_, ns // 3)) + 0.25 if ns >= 3 else short[: ns // 3]
    short.sort()
    for diff, off in ((0.25, 0.0), (0.01, 0.0105), (0.25, -0.125)):
        got = _kernel_assoc(long_, short, diff, off)                      # e shorter: offset applies to r, negated
        want = O.associate(long_, short, diff, off)[:2]
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
    # huge stamps: all differences round alike and the lowest index wins
    big = np.full(7, 1311868160.0)
    np.testing.assert_array_equal(_kernel_assoc(big[:3], big[:5], 1.0, 0.0), O.associate(big[:3], big[:5], 1.0, 0.0)[:2])


@pytest.mark.gpu
def test_caller_stamps_are_not_modified():
    rs = torch.arange(100, dtype=torch.float64, device=DEV)
    es = torch.arange(50, dtype=torch.float64, device=DEV) * 2 + 0.5
    keep = (rs.clone(), es.clone())
    P = pp.randn_SE3(100, device=DEV, dtype=torch.float64)
    pp.metric.ape(rs, P, es, P[:50], offset=0.5, diff=0.1)
    pp.metric.ape(es, P[:50], rs, P, offset=0.5, diff=0.1)
    assert torch.equal(rs, keep[0]) and torch.equal(es, keep[1])
    with pytest.raises(ValueError):
        pp.metric.ape(rs[:3], P, es, P[:50])                        # stamps and poses of different lengths
    with pytest.raises(ValueError):
        pp.metric.ape(rs.flip(0), P, es, P[:50])                    # unsorted stamps
    with pytest.raises(ValueError):
        pp.metric.ape(rs, P, es + 1000, P[:50])                     # no match
    with pytest.raises(ValueError):
        pp.metric.rpe(rs, P, es, P[:50], offset=0.5, diff=0.1, delta=100)   # no pair


def _path(n, g, plateau=True):
    step = g.normal(size=(n, 3)) * 0.05 + [0.03, 0.01, 0.0]
    if plateau:
        step[(np.arange(n) // 5) % 4 == 0] = 0.0
    step[0] = 0.0
    t = np.cumsum(step, 0)
    q = g.normal(size=(n, 4)) * 0.1 + [0.0, 0.0, 0.0, 1.0]
    return np.concatenate([t, q / np.linalg.norm(q, axis=-1, keepdims=True)], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 2047, 2048, 2049, 4097, 10**6])
@pytest.mark.parametrize("all_", [False, True])
def test_distance_pairs_equal_oracle(n, all_):
    g = np.random.default_rng(n)
    P = _path(n, g)
    idx = torch.arange(n, device=DEV)
    for dtype in (torch.float64, torch.float32):
        Pd = torch.from_numpy(P).to(DEV, dtype)
        Pw = Pd.double().cpu().numpy()
        for delta in (0.3, 2.0):
            src, tgt = A._pairs_by_dist(Pd, idx, None, delta, delta * 0.1, all_)
            osrc, otgt = O.pairs_by_dist(Pw[:, :3], delta, delta * 0.1, all_)
            np.testing.assert_array_equal(src.cpu().numpy(), osrc)
            np.testing.assert_array_equal(tgt.cpu().numpy(), otgt)


@pytest.mark.gpu
@pytest.mark.parametrize("etype", O.ETYPES)
def test_errors_equal_oracle(etype):
    g = np.random.default_rng(5)
    n = 20000
    P = [_path(n, g, False) for _ in range(2)]
    P[1][:, 3:] = P[1][:, 3:].astype(np.float32)         # non-unit fp32 quaternions
    S = np.array([0.3, -0.2, 1.0, 0.1, -0.2, 0.3, 0.9273618495495703, 1.3])
    S[3:7] /= np.linalg.norm(S[3:7])
    ra = np.sort(g.integers(0, n, 5000))
    rb = np.minimum(ra + 3, n - 1)
    ti = lambda a: torch.from_numpy(a).to(DEV)          # noqa: E731
    for s in (None, S):
        St = None if s is None else ti(s)
        e = A._errors(ti(P[0]), ti(P[1]), ti(ra), None, ti(ra), None, St, etype).cpu().numpy()
        assert close(e, O.ape_errors(P[0][ra], O.align(s, P[1][ra]), etype))
        e = A._errors(ti(P[0]), ti(P[1]), ti(ra), ti(rb), ti(ra), ti(rb), St, etype).cpu().numpy()
        assert close(e, O.rpe_errors(P[0][ra], P[0][rb], O.align(s, P[1][ra]), O.align(s, P[1][rb]), etype))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2, 3, 255, 256, 257, 2047, 2048, 2049, 2048 * 1024 - 1, 2048 * 1024 + 1, 10**7])
def test_statistics(M):
    g = np.random.default_rng(M)
    for kind in ("rand", "equal", "zeros"):
        e = g.gamma(2.0, size=M) if kind == "rand" else np.full(M, 0.7) if kind == "equal" else np.zeros(M)
        if kind != "rand" and M > 2049:
            continue
        et = torch.from_numpy(e).to(DEV)
        out = A._statistics(et, "All")
        want = O.stats(e)
        srt = np.sort(e)
        assert out["Max"].item() == srt[-1] and out["Min"].item() == srt[0]
        assert out["Median"].item() == srt[(M - 1) // 2]
        for k in ("Mean", "RMSE", "SSE", "STD"):
            assert close(out[k].item(), want[k]), (k, out[k].item(), want[k])
        if M == 1:
            assert math.isnan(out["STD"].item())
        for k in O.KEYS:                                  # one statistic alone is the same value
            assert A._statistics(et, k).item() == out[k].item() or (k == "STD" and M == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("fn,kw", [("ape", dict(etype="pose")), ("ape", dict(etype="degree", align=True, scale=True)),
                                   ("rpe", dict(associate="distance", delta=0.5, all=True)),
                                   ("rpe", dict(associate="distance", delta=0.5, rpair=True)),
                                   ("rpe", dict(etype="radian", delta=2, origin=True))])
def test_fp32_strided_and_repeatable(fn, kw):
    g = np.random.default_rng(9)
    n = 30000
    P, E = _path(n, g), _path(n, g)
    rs, es = np.arange(n) * 0.01, np.arange(n // 2) * 0.02 + 0.001
    f32 = run_metric(fn, rs, P, es, E[: n // 2], kw, torch.float32)
    Pw, Ew = P.astype(np.float32).astype(np.float64), E[: n // 2].astype(np.float32).astype(np.float64)
    f64 = run_metric(fn, rs, Pw, es, Ew, kw)
    again = run_metric(fn, rs, Pw, es, Ew, kw)
    # a strided view: every other row of a wider buffer, columns at stride 2
    big = torch.zeros(2 * n, 14, dtype=torch.float64, device=DEV)
    big[::2, ::2] = torch.from_numpy(Pw).to(DEV)
    strided = pp.metric.__dict__[fn](torch.from_numpy(rs).to(DEV), pp.SE3(big[::2, ::2]), torch.from_numpy(es).to(DEV),
                                     pp.SE3(torch.from_numpy(Ew).to(DEV)), **kw)
    for k in O.KEYS:
        a = f32[k].item()
        assert a == f64[k].item() == again[k].item() == strided[k].item() or (math.isnan(a) and math.isnan(f64[k].item()))


@pytest.mark.gpu
@pytest.mark.parametrize("fn,kw,reads", [("ape", {}, 1), ("rpe", {}, 1), ("rpe", dict(all=True, delta=3), 1),
                                         ("rpe", dict(associate="distance", delta=0.5), 2),
                                         ("rpe", dict(associate="distance", delta=0.5, all=True), 2)])
def test_host_read_budget(fn, kw, reads):
    g = np.random.default_rng(2)
    n = 5000
    args = [torch.from_numpy(a).to(DEV) for a in (np.arange(n) * 0.01, _path(n, g), np.arange(n) * 0.01, _path(n, g))]
    args[1], args[3] = pp.SE3(args[1]), pp.SE3(args[3])
    getattr(pp.metric, fn)(*args, **kw)                 # warm up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            getattr(pp.metric, fn)(*args, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) == reads, [str(x.message) for x in syncs]
