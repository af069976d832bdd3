"""Every launch path of csrc/lqr.cu against an fp64 dense-KKT oracle (oracle/lqr_kkt.py), in fp32 and fp64.

The kernels run one problem per warp and put w = 1..8 warps in a CTA, each on its own slab of `lqr_smem_elems(ns, nc)`
elements of dynamic shared memory: w = 48 KB / slab bytes, clamped to [1, 8] (DESIGN.md §3.7).  `warps` mirrors that
rule; the mirror is checked against the host build of lqr_math.cuh (tests/lqr_host.cpp) and against the launches the
profiler records, and every GPU test asserts the w its shape reaches.  The shapes cover w = 1..8 in fp64 and w = 2..8 in
fp32 (no fp32 shape with n <= 32 needs a whole CTA); batches of 2w + 1 problems leave the last CTA ragged.

Tolerances: fp64 1e-10 relative against the oracle for every problem, 1e-9 for gradients; fp32: the worst problem within
4x the worst error of the generic route (the reference's algorithm in torch ops) run in fp32 on the CPU with the same
inputs.  That bound is never tighter than 4x the larger of 4 ulps and n u (u = 2^-24, n = ns + nc), the rounding bound
of one length-n dot product accumulated in order, as the kernel does: where both routes are exact to a few ulps the
ratio of two errors is noise.  Errors are relative to the largest element of each problem.  A gradient is compared
relative to its own largest element, or to 1e-3 of the largest element of all six gradients when it is smaller (a
gradient that is zero in exact arithmetic, such as that of c1_{T-1} when x_T gets no cotangent, is then not compared
with rounding noise).
"""
import ctypes
import functools
import json
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import lqr_kkt as K
from oracle import lqr_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
F32, F64 = torch.float32, torch.float64
BUDGET = 48 * 1024
TS = (1, 2, 17)
KEYS = ("Q", "p", "A", "B", "c1", "x0")
FLOOR32 = 2.0 ** -21                   # 4 ulps of fp32

# (ns, nc) per warps-per-CTA and dtype
W_SHAPES = {
    F64: {1: ((31, 1), (20, 12)), 2: ((1, 31), (16, 16)), 3: ((17, 3),), 4: ((15, 3),), 5: ((14, 2),), 6: ((12, 4),),
          7: ((10, 5),), 8: ((4, 3), (1, 1))},
    F32: {2: ((31, 1),), 3: ((27, 5), (20, 12)), 4: ((16, 16),), 5: ((1, 31),), 6: ((19, 2),), 7: ((17, 3),),
          8: ((4, 3), (12, 4))},
}
CASES = [(dt, w, s) for dt in (F64, F32) for w, ss in W_SHAPES[dt].items() for s in ss]
SHAPES = sorted({s for _, _, s in CASES})


def _dn(dt):
    return "f64" if dt == F64 else "f32"


def _cid(c):
    return f"{_dn(c[0])}-w{c[1]}-{c[2][0]}x{c[2][1]}"


def slab_elems(ns, nc):
    """lqr_smem_elems of csrc/lqr_math.cuh"""
    n = ns + nc
    e = n * n + 2 * n * ns + ns * ns + nc * nc + nc * (ns + 1) + 4 * n + 3 * ns
    return (e + 1) & ~1


def warps(ns, nc, dtype):
    """warps_per_cta of csrc/lqr.cu"""
    w = BUDGET // (slab_elems(ns, nc) * (4 if dtype == F32 else 8))
    return min(max(w, 1), 8)


def _seed(*key):
    return zlib.crc32(repr(key).encode())


@functools.lru_cache(maxsize=None)
def _problem(nb, T, ns, nc, seed, lti):
    g = torch.Generator().manual_seed(seed)
    n = ns + nc
    r = lambda *s: torch.randn(*s, generator=g, dtype=F64)   # noqa: E731
    M = r(nb, T, n, n)
    Q = M.mT @ M / n + torch.eye(n, dtype=F64)
    Q = 0.5 * (Q + Q.mT)
    Tm = 1 if lti else T
    A = 0.8 * torch.eye(ns, dtype=F64) + 0.2 / ns ** 0.5 * r(nb, Tm, ns, ns)
    B, c1 = r(nb, Tm, ns, nc) / nc ** 0.5, r(nb, Tm, ns)
    A, B, c1 = (t.expand(nb, T, *t.shape[2:]).contiguous() for t in (A, B, c1))
    return dict(Q=Q, p=r(nb, T, n), A=A, B=B, c1=c1, x0=r(nb, ns), u=r(nb, T, nc))


def problem(nb, T, ns, nc, seed, lti=False):
    """a well-conditioned random fp64 problem on the CPU, every operand at full size (nb, T, ...): Q symmetric positive
    definite, A_t near 0.8 I; lti: A, B and c1 the same at every step"""
    return {k: v.clone() for k, v in _problem(nb, T, ns, nc, seed, lti).items()}


def cotangents(nb, T, ns, nc, seed):
    g = torch.Generator().manual_seed(seed + 1)
    return (torch.randn(nb, T + 1, ns, generator=g, dtype=F64), torch.randn(nb, T, nc, generator=g, dtype=F64),
            torch.randn(nb, generator=g, dtype=F64))


def oracle(P, T):
    """-> x, u, cost, x_traj of the KKT oracle (fp64, CPU)"""
    with torch.no_grad():
        x, u, c = K.solve(P["Q"], P["p"], P["A"], P["B"], P["c1"], P["x0"], T)
        return x, u, c, K.rollout(P["A"], P["B"], P["c1"], P["x0"], P.get("u"), T)


def relb(a, b):
    """per-problem relative error: max |a - b| over max |b| of each problem (leading axis)"""
    a, b = (torch.as_tensor(t).detach().cpu().double().reshape(t.shape[0], -1) for t in (a, b))
    return ((a - b).abs().amax(1) / b.abs().amax(1).clamp_min(1e-300)).numpy()


def sym(g):
    return 0.5 * (g + g.mT)


def grad_errs(got, want):
    """per operand: max |got - want| over max(max |want|, 1e-3 * max over all the wanted gradients); Q symmetrised"""
    scale = max(float(w.abs().max()) for w in want.values())
    out = {}
    for k, w in want.items():
        g = got[k].detach().cpu().double().reshape(w.shape)
        if k == "Q":
            g, w = sym(g), sym(w)
        out[k] = float((g - w).abs().max()) / max(float(w.abs().max()), 1e-3 * scale, 1e-300)
    return out


def check(err, ref, dtype, tol64, what, n):
    """fp64: every err <= tol64; fp32: max err <= 4 * max(max ref, 2^-21, n 2^-24), ref the fp32 generic route's
    errors, n = ns + nc"""
    err = np.asarray(err)
    lim = tol64 if dtype == F64 else 4 * max(float(np.max(ref)), FLOOR32, n * 2.0 ** -24)
    assert np.all(err <= lim), (what, err, lim)


# ------------------------------------------------------------------------------------------------- systems and runs
class StepLTV(pp.module.LTV):
    """A_t, B_t and c1_t read at the system time: the affine route gathers them per step ('gather')"""
    @property
    def A(self):
        return self._A[:, int(self._t)]

    @property
    def B(self):
        return self._B[:, int(self._t)]

    @property
    def c1(self):
        return self._c1[:, int(self._t)]


def module(P, T, dtype, device, kind, u=True):
    """pp.module.LQR on P: kind 'step' (StepLTV, per-step A, B, c1), 'lti' or 'ltv' (P's step-0 A, B, c1 through
    pp.module.LTI / pp.module.LTV).  -> (lqr, leaves requiring grad, (x, u, cost)); the generic route on the CPU."""
    nb, ns = P["x0"].shape
    nc = P["B"].shape[-1]
    ins = {k: (P[k][:, 0] if kind != "step" and k in ("A", "B", "c1") else P[k]).to(device, dtype).clone()
           for k in KEYS}
    ins = {k: v.requires_grad_() for k, v in ins.items()}
    C = torch.eye(ns, dtype=dtype, device=device).expand(nb, ns, ns)
    D = torch.zeros(nb, ns, nc, dtype=dtype, device=device)
    cls = {"step": StepLTV, "lti": pp.module.LTI, "ltv": pp.module.LTV}[kind]
    lqr = pp.module.LQR(cls(ins["A"], ins["B"], C, D, ins["c1"]), ins["Q"], ins["p"], T)
    ut = P["u"].to(device, dtype) if u else None
    if device == DEV:
        assert lqr._route(ins["x0"], 1, ut) == {"step": "gather", "lti": "lti", "ltv": "ltv"}[kind]
    return lqr, ins, lqr(ins["x0"], 1, ut)


def run(P, dtype, T, grad=False):
    """torch.ops.b200pose.lqr_affine on P's operands as given (c1 / u may be None) -> (leaves, outputs)"""
    ins = {k: None if P.get(k) is None else P[k].to(DEV, dtype).clone() for k in KEYS + ("u",)}
    for k in KEYS:
        if grad and ins[k] is not None:
            ins[k].requires_grad_()
    out = torch.ops.b200pose.lqr_affine(ins["Q"], ins["p"], ins["A"], ins["B"], ins["c1"], ins["x0"], ins["u"], T)
    return ins, out


SUBSETS = ("cost", "x", "xT", "u", "all")


def pick(subset, x, u, cost, cot, T):
    """outputs and cotangents of one cotangent subset; outputs left out get no gradient (None in the backward)"""
    gx, gu, gc = (c.to(x.device, x.dtype) for c in cot)
    return {"cost": ([cost], [gc]), "x": ([x], [gx]), "xT": ([x[:, T]], [gx[:, T]]), "u": ([u], [gu]),
            "all": ([x, u, cost], [gx, gu, gc])}[subset]


def grads(ins, outs, subset, cot, T, keys=KEYS):
    o, g = pick(subset, *outs, cot, T)
    keys = [k for k in keys if ins.get(k) is not None]
    gs = torch.autograd.grad(o, [ins[k] for k in keys], g, retain_graph=True, allow_unused=True)
    return {k: torch.zeros_like(ins[k]) if v is None else v for k, v in zip(keys, gs)}   # the generic route at T = 1


# ------------------------------------------------------------------------------------------------------------- CPU
_HOST = {}


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="lqr_paths_host_")
        so = os.path.join(d, "liblqrhost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "lqr_host.cpp"),
                               "-o", so])
        lib = ctypes.CDLL(so)
        lib.lqr_host_smem_elems.restype, lib.lqr_host_smem_elems.argtypes = ctypes.c_int, [ctypes.c_int, ctypes.c_int]
        _HOST["lib"] = lib
    return _HOST["lib"]


def test_mirror_matches_host_build():
    pairs = [(ns, n - ns) for n in range(2, 33) for ns in range(1, n)]
    assert len(pairs) == 496
    for ns, nc in pairs:
        assert slab_elems(ns, nc) == _host().lqr_host_smem_elems(ns, nc), (ns, nc)
    for dt, w, (ns, nc) in CASES:
        assert warps(ns, nc, dt) == w, (dt, ns, nc)
    assert sorted({w for dt, w, _ in CASES if dt == F64}) == list(range(1, 9))
    assert sorted({w for dt, w, _ in CASES if dt == F32}) == list(range(2, 9))
    assert min(warps(ns, n - ns, F32) for n in range(2, 33) for ns in range(1, n)) == 2


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_kkt_matches_riccati_oracle(shape, T):
    """the KKT oracle and the restatement of the kernel's algorithm (oracle/lqr_oracle.py) agree"""
    ns, nc = shape
    P = problem(2, T, ns, nc, _seed("cpu", shape, T))
    ins = {k: P[k].clone().requires_grad_() for k in KEYS}
    x, u, c = K.solve(*[ins[k] for k in KEYS], T)
    F = [P[k].numpy() for k in KEYS + ("u",)]
    xo, uo, co, xto, st = O.lqr(*F)
    assert not st.any() and not K.status(P["Q"], P["A"], P["B"], 2, T).any()
    for a, b in ((x, xo), (u, uo), (c, co), (K.rollout(P["A"], P["B"], P["c1"], P["x0"], P["u"], T), xto)):
        assert relb(a, torch.from_numpy(b)).max() < 1e-10
    cot = cotangents(2, T, ns, nc, 0)
    got = dict(zip(KEYS, torch.autograd.grad((x * cot[0]).sum() + (u * cot[1]).sum() + (c * cot[2]).sum(),
                                             [ins[k] for k in KEYS])))
    want = O.lqr_bwd(*F[:6], xo, uo, *(t.numpy() for t in cot))
    errs = grad_errs(got, {k: torch.from_numpy(w) for k, w in zip(KEYS, want)})
    assert max(errs.values()) < 1e-10, errs


GOLD = np.load(os.path.join(ROOT, "tests", "golden", "lqr.npz"))
GCASES = json.loads(str(GOLD["cases"]))


@pytest.mark.parametrize("name", [k for k, c in GCASES.items()
                                  if c["kind"] in ("lti", "ltv") and not c["raises"] and c["dt"] == 1])
def test_kkt_matches_reference_goldens(name):
    c = GCASES[name]
    g = lambda k: None if f"{name}/{k}" not in GOLD.files else torch.from_numpy(GOLD[f"{name}/{k}"])   # noqa: E731
    T = c["T"]
    ins = {"Q": g("Q"), "p": g("p"), "A": g("A"), "B": g("B"), "c1": g("c1"), "x0": g("x0")}
    ins = {k: None if v is None else v.clone().requires_grad_() for k, v in ins.items()}
    step = {"Q": 4, "p": 3, "A": 4, "B": 4, "c1": 3}   # ndim of an operand with a step axis
    ops = {k: None if v is None else (v if v.ndim == step[k] else v[:, None]) for k, v in ins.items() if k != "x0"}
    x, u, cost = K.solve(ops["Q"], ops["p"], ops["A"], ops["B"], ops["c1"], ins["x0"], T)
    for a, k in ((x, "x"), (u, "u"), (cost, "cost")):
        assert relb(a, g(k)).max() < 1e-10, k
    if c["grad"]:
        keys = [k for k in KEYS if ins[k] is not None]
        gr = torch.autograd.grad((x * g("gx")).sum() + (u * g("gu")).sum() + (cost * g("gc")).sum(),
                                 [ins[k] for k in keys])
        errs = grad_errs(dict(zip(keys, gr)), {k: g(f"g{k}") for k in keys})
        assert max(errs.values()) < 1e-9, errs


BAD = ("indefinite", "fvf", "singular", "nan")


def make_bad(P, b, kind, T):
    """problem b of P made one that the Riccati recursion cannot solve:
    indefinite: its own Quu at t = T-1 (the first step processed);
    fvf: every Q_t uu block positive definite, but Quu at t = 0 indefinite through F^T V F (a very negative Qxx at t = 1);
    singular: Quu at t = T-1 exactly singular (its last row and column 0);
    nan: one NaN in the lower triangle of Quu (the diagonal when nc = 1) at t = 2."""
    ns = P["x0"].shape[1]
    n = P["p"].shape[-1]
    nc = n - ns
    Q = P["Q"]
    if kind == "indefinite":
        Q[b, T - 1, ns:, ns:] -= 1e3 * torch.eye(nc, dtype=Q.dtype)
    elif kind == "fvf":
        Q[b, 1, :ns, :ns] -= 1e3 * torch.eye(ns, dtype=Q.dtype)
    elif kind == "singular":
        Q[b, T - 1, n - 1, :] = 0
        Q[b, T - 1, :, n - 1] = 0
    else:
        Q[b, 2, n - 1, ns] = float("nan")


@pytest.mark.parametrize("kind", BAD)
def test_status_oracle_agrees_with_riccati_oracle(kind):
    T, ns, nc = 4, 4, 3
    P = problem(3, T, ns, nc, _seed("status", kind))
    make_bad(P, 1, kind, T)
    st = K.status(P["Q"], P["A"], P["B"], 3, T)
    assert st.tolist() == [0, 1, 0]
    F = [np.ascontiguousarray(P[k].numpy()) for k in KEYS + ("u",)]
    if kind != "nan":                   # numpy's cholesky does not reject a NaN
        assert np.array_equal(O.lqr(*F)[4], st.numpy())
    x, u, cost, xt = np.empty((3, T + 1, ns)), np.empty((3, T, nc)), np.empty(3), np.empty((3, T, ns))
    hst = np.empty(3, np.int32)
    _host().lqr_host_solve(*[ctypes.c_void_p(a.ctypes.data) for a in F], ctypes.c_longlong(3), T, ns, nc,
                           *[ctypes.c_void_p(a.ctypes.data) for a in (x, u, cost, xt, hst)])
    assert np.array_equal(hst, st.numpy())


# ------------------------------------------------------------------------------------------------------------- GPU
def generic32(P, T, kind="step", u=True):
    """the fp32 generic route on the CPU: (lqr, leaves, (x, u, cost))"""
    return module(P, T, F32, "cpu", kind, u)


def _fwd_errs(got, want):
    return [relb(g, w) for g, w in zip(got, want)]


@pytest.mark.gpu
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_every_w_every_slot(case, T):
    """x, u, cost and x_traj of every problem of a batch of 2w + 1 (ragged last CTA) and of w - 1 (one partial CTA)"""
    dt, w, (ns, nc) = case
    assert warps(ns, nc, dt) == w
    for nb in sorted({2 * w + 1, w - 1} - {0}):
        P = problem(nb, T, ns, nc, _seed("slot", case[1:], T, nb))
        _, (x, u, cost, xtr, st) = run(P, dt, T)
        assert not st.any()
        want = oracle(P, T)
        ref = None
        if dt == F32:
            lqr, _, r = generic32(P, T)
            ref = _fwd_errs((*r, lqr.x_traj), want)
        for i, (got, wnt, name) in enumerate(zip((x, u, cost, xtr), want, ("x", "u", "cost", "x_traj"))):
            check(relb(got, wnt), None if ref is None else ref[i], dt, 1e-10, (name, nb), ns + nc)


@pytest.mark.gpu
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_slot_invariance_bit_for_bit(case, T):
    """each problem of a 2w + 1 batch solved alone gives the same bits, forward and all six gradients"""
    dt, w, (ns, nc) = case
    assert warps(ns, nc, dt) == w
    nb = 2 * w + 1
    P = problem(nb, T, ns, nc, _seed("inv", case[1:], T))
    cot = cotangents(nb, T, ns, nc, 7)
    ins, out = run(P, dt, T, grad=True)
    g = grads(ins, out[:3], "all", cot, T)
    for b in range(nb):
        Pb = {k: v[b:b + 1] for k, v in P.items()}
        ib, ob = run(Pb, dt, T, grad=True)
        gb = grads(ib, ob[:3], "all", tuple(c[b:b + 1] for c in cot), T)
        for s, t in zip(out, ob):
            assert torch.equal(s[b:b + 1], t), b
        for k in KEYS:
            assert torch.equal(g[k][b:b + 1], gb[k]), (b, k)


def _placements(nb, T):
    return {"11": (1, 1), "n1": (nb, 1), "1T": (1, T)}


BCAST = [(k, pl) for k in ("Q", "p", "A", "B", "c1", "u") for pl in ("11", "n1", "1T")] + \
        [("all", "11"), ("none", "nT"), ("c1", "None"), ("u", "None")]
BSHAPES = [(F64, 8, (4, 3)), (F64, 1, (31, 1)), (F32, 8, (12, 4)), (F32, 2, (31, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("bc", BCAST, ids=lambda b: f"{b[0]}-{b[1]}")
@pytest.mark.parametrize("case", BSHAPES, ids=_cid)
def test_broadcast_operands(case, bc):
    """an operand broadcast over the batch and / or the steps (zero strides) against the same operand materialised:
    the forward is bit-identical; its gradient is the materialised per-step gradients summed over the broadcast axes"""
    dt, w, (ns, nc) = case
    assert warps(ns, nc, dt) == w
    T, nb = 5, 2 * w + 1
    P = problem(nb, T, ns, nc, _seed("bcast", case[1:], bc))
    name, pl = bc
    compact = dict(P)
    if pl == "None":
        compact[name] = None
    elif pl != "nT":
        sn, st = _placements(nb, T)[pl]
        for k in (("Q", "p", "A", "B", "c1", "u") if name == "all" else (name,)):
            compact[k] = P[k][:sn, :st].contiguous()
    mat = {k: v if k == "x0" else torch.zeros_like(P[k]) if v is None else v.expand(nb, T, *v.shape[2:]).contiguous()
           for k, v in compact.items()}
    cot = cotangents(nb, T, ns, nc, 3)
    ic, oc = run(compact, dt, T, grad=True)
    im, om = run(mat, dt, T, grad=True)
    for s, t in zip(oc, om):
        assert torch.equal(s, t)
    gc, gm = grads(ic, oc[:3], "all", cot, T), grads(im, om[:3], "all", cot, T)
    want = {}
    for k, g in gc.items():
        dims = tuple(d for d in (0, 1) if ic[k].shape[d] == 1 and k != "x0")
        want[k] = (gm[k].sum(dims, keepdim=True) if dims else gm[k]).double().cpu()
        assert g.shape == ic[k].shape
    errs = grad_errs(gc, want)
    assert max(errs.values()) <= (1e-12 if dt == F64 else 3e-5), errs


@pytest.mark.gpu
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_adjoint_against_kkt_autograd(case, T):
    """the six gradients through lqr_affine, LQR on a per-step LTV ('gather'), an LTI and an LTV, for the cotangents of
    cost, x, x_T, u or all three, against autograd through the KKT solve"""
    dt, w, (ns, nc) = case
    assert warps(ns, nc, dt) == w
    nb = 2 * w + 1
    for lti in (False, True):
        P = problem(nb, T, ns, nc, _seed("adj", case[1:], T), lti=lti)
        cot = cotangents(nb, T, ns, nc, 11)
        kin = {k: (P[k][:, :1] if lti and k in ("A", "B", "c1") else P[k]).clone().requires_grad_() for k in KEYS}
        kout = K.solve(*[kin[k] for k in KEYS], T)
        runs = {}
        if lti:
            for kind in ("lti", "ltv"):
                _, i, o = module(P, T, dt, DEV, kind)
                runs[kind] = (i, o)
        else:
            i, o = run(P, dt, T, grad=True)
            runs["op"] = (i, o[:3])
            _, i, o = module(P, T, dt, DEV, "step")
            runs["gather"] = (i, o)
        ref = generic32(P, T, "lti" if lti else "step") if dt == F32 else None
        for subset in SUBSETS:
            want = {k: v.detach() for k, v in grads(kin, kout, subset, cot, T).items()}
            rerr = None if ref is None else grad_errs(grads(ref[1], ref[2], subset, cot, T), want)
            for entry, (i, o) in runs.items():
                errs = grad_errs(grads(i, o, subset, cot, T), want)
                for k in KEYS:
                    check(errs[k], None if rerr is None else rerr[k], dt, 1e-9, (entry, subset, k), ns + nc)


STATUS = [(F64, 1, (31, 1)), (F64, 2, (16, 16)), (F64, 8, (4, 3)), (F32, 2, (31, 1)), (F32, 8, (4, 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", BAD)
@pytest.mark.parametrize("case", STATUS, ids=_cid)
def test_status_per_problem(case, kind):
    """bad problems in the first, a middle and the last warp slot: the status equals the oracle's per problem, the good
    problems' outputs are bit-identical to a batch without the bad ones, and LQR raises"""
    dt, w, (ns, nc) = case
    assert warps(ns, nc, dt) == w
    T, nb = 4, 2 * w + 1
    bad = sorted({0, w + w // 2, 2 * w - 1}) if w > 1 else [0, 2]
    P = problem(nb, T, ns, nc, _seed("status", case[1:], kind))
    for b in bad:
        make_bad(P, b, kind, T)
    want = K.status(P["Q"], P["A"], P["B"], nb, T)
    assert want.nonzero().flatten().tolist() == bad
    _, (x, u, cost, xtr, st) = run(P, dt, T)
    assert torch.equal(st.cpu(), want)
    good = [b for b in range(nb) if b not in bad]
    _, ref = run({k: v[good] for k, v in P.items()}, dt, T)
    assert not ref[4].any()
    for s, t in zip((x, u, cost, xtr), ref[:4]):
        assert torch.equal(s[good], t)
    with pytest.raises(torch.linalg.LinAlgError):
        module(P, T, dt, DEV, "step")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in STATUS if c[1] > 1], ids=_cid)
def test_adjoint_isolated_from_failing_neighbours(case):
    """lqr_affine_bwd on a batch whose even problems have an indefinite Q_t uu at every step: the Cholesky of those warps
    fails at once at every step, so they run ahead of their neighbours in the same CTA and reach the last pass (lam,
    dlam) while the odd problems still run the recursion (Qt, at the start of the next warp's slab).  The odd problems'
    gradients are bit-identical to a batch of the odd problems alone."""
    dt, w, (ns, nc) = case
    assert warps(ns, nc, dt) == w
    T, nb = 64, 2 * w + 1
    P = problem(nb, T, ns, nc, _seed("isolated", case[1:]))
    bad, good = list(range(0, nb, 2)), list(range(1, nb, 2))
    P["Q"][bad, :, ns:, ns:] -= 1e3 * torch.eye(nc, dtype=F64)
    _, (x, u, _, _, st) = run(P, dt, T)
    assert st.cpu().tolist() == [1, 0] * w + [1]
    x[bad], u[bad] = 0, 0
    gx, gu, gc = (c.to(DEV, dt) for c in cotangents(nb, T, ns, nc, 13))
    ins = {k: P[k].to(DEV, dt) for k in KEYS}
    g = torch.ops.b200pose.lqr_affine_bwd(*[ins[k] for k in KEYS], T, x, u, gx, gu, gc)
    P = {k: v[good] for k, v in P.items()}
    ins, (xg, ug, _, _, st) = run(P, dt, T)
    assert not st.any() and torch.equal(xg, x[good]) and torch.equal(ug, u[good])
    want = torch.ops.b200pose.lqr_affine_bwd(*[ins[k] for k in KEYS], T, xg, ug, gx[good], gu[good], gc[good])
    for k, a, b in zip(KEYS, g, want):
        assert torch.equal(a[good], b), k


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (F64, F32), ids=_dn)
def test_one_million_problems(dt):
    """nb = 2^20 + 3 at (1, 1), T = 4: a sample of problems, the last CTA (3 problems) and the one before it"""
    ns, nc, T = 1, 1, 4
    nb = 2 ** 20 + 3
    assert warps(ns, nc, dt) == 8 and nb % 8 == 3
    g = torch.Generator().manual_seed(21)
    r = lambda *s: torch.randn(*s, generator=g, dtype=F64)   # noqa: E731
    M = r(nb, T, 2, 2)
    P = dict(Q=sym(M.mT @ M / 2 + torch.eye(2, dtype=F64)), p=r(nb, T, 2), A=0.8 + 0.2 * r(nb, T, 1, 1),
             B=r(nb, T, 1, 1), c1=r(nb, T, 1), x0=r(nb, 1), u=r(nb, T, 1))
    _, out = run(P, dt, T)
    assert not out[4].any()
    idx = torch.from_numpy(np.unique(np.r_[np.random.default_rng(0).choice(nb, 64, replace=False),
                                           np.arange(nb - 11, nb), 0, 1]))
    S = {k: v[idx] for k, v in P.items()}
    want = oracle(S, T)
    ref = None
    if dt == F32:
        lqr, _, rr = generic32(S, T)
        ref = _fwd_errs((*rr, lqr.x_traj), want)
    for i, (a, b) in enumerate(zip(out[:4], want)):
        check(relb(a[idx.to(DEV)], b), None if ref is None else ref[i], dt, 1e-10, i, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (F64, F32), ids=_dn)
def test_long_horizon(dt):
    """T = 1000 at (4, 3) against the Riccati oracle"""
    ns, nc, T = 4, 3, 1000
    nb = 2 * warps(ns, nc, dt) + 1
    P = problem(nb, T, ns, nc, _seed("long"))
    _, (x, u, cost, xtr, st) = run(P, dt, T)
    assert not st.any()
    want = [torch.from_numpy(a) for a in O.lqr(*[P[k].numpy() for k in KEYS + ("u",)])[:4]]
    ref = None
    if dt == F32:
        lqr, _, rr = generic32(P, T)
        ref = _fwd_errs((rr[0], rr[1], rr[2][:, None], lqr.x_traj), (want[0], want[1], want[2][:, None], want[3]))
    for i, (a, b) in enumerate(zip((x, u, cost[:, None], xtr), (want[0], want[1], want[2][:, None], want[3]))):
        check(relb(a, b), None if ref is None else ref[i], dt, 1e-10, i, ns + nc)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (F64, F32), ids=_dn)
def test_gather_route(dt):
    """an LTV subclass with per-step A, B, c1 properties at (16, 16), T = 20: forward and gradients"""
    ns, nc, T = 16, 16, 20
    w = warps(ns, nc, dt)
    assert w == (2 if dt == F64 else 4)
    nb = 2 * w + 1
    P = problem(nb, T, ns, nc, _seed("gather"))
    cot = cotangents(nb, T, ns, nc, 5)
    lqr, ins, out = module(P, T, dt, DEV, "step")
    kin = {k: P[k].clone().requires_grad_() for k in KEYS}
    kout = K.solve(*[kin[k] for k in KEYS], T)
    want = oracle(P, T)
    ref = rerr = None
    if dt == F32:
        rl, ri, ro = generic32(P, T)
        ref = _fwd_errs((*ro, rl.x_traj), want)
    for i, (a, b) in enumerate(zip((*out, lqr.x_traj), want)):
        check(relb(a.reshape(nb, -1), b.reshape(nb, -1)), None if ref is None else ref[i], dt, 1e-10, i, ns + nc)
    kg = {k: v.detach() for k, v in grads(kin, kout, "all", cot, T).items()}
    if dt == F32:
        rerr = grad_errs(grads(ri, ro, "all", cot, T), kg)
    errs = grad_errs(grads(ins, out, "all", cot, T), kg)
    for k in KEYS:
        check(errs[k], None if rerr is None else rerr[k], dt, 1e-9, k, ns + nc)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (F64, F32), ids=_dn)
def test_mpc_on_lti_equals_one_affine_solve(dt):
    """MPC on an LTI at n = 32: every pass runs the affine route and the result is the one minimiser"""
    ns, nc, T = 20, 12, 10
    P = problem(1, T, ns, nc, _seed("mpc"), lti=True)
    C, D = torch.eye(ns, dtype=dt, device=DEV)[None], torch.zeros(1, ns, nc, dtype=dt, device=DEV)
    dev = {k: P[k].to(DEV, dt) for k in KEYS}
    lti = pp.module.LTI(dev["A"][:, 0], dev["B"][:, 0], C, D, dev["c1"][:, 0])
    x, u, cost = pp.module.MPC(lti, dev["Q"], dev["p"], T, stepper=pp.utils.ReduceToBason(3))(1, dev["x0"])
    _, one = run({**P, "A": P["A"][:, :1], "B": P["B"][:, :1], "c1": P["c1"][:, :1], "u": None}, dt, T)
    want = oracle({**P, "u": None}, T)
    ref = [np.zeros(1)] * 3
    if dt == F32:
        ref = _fwd_errs(generic32(P, T, "lti", u=False)[2], want[:3])
    for i, (a, b, c) in enumerate(zip((x, u, cost[:, None]), one[:3], (want[0], want[1], want[2][:, None]))):
        check(relb(a, c), ref[i], dt, 1e-10, ("mpc", i), ns + nc)
        check(relb(b.reshape(a.shape), c), ref[i], dt, 1e-10, ("affine", i), ns + nc)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (F64, F32), ids=_dn)
def test_launch_shape_is_the_mirrored_one(dt, tmp_path):
    """the profiler's record of each forward and backward launch: 32 w threads per CTA and ceil(nb / w) CTAs"""
    for case in [c for c in CASES if c[0] == dt]:
        _, w, (ns, nc) = case
        nb, T = 2 * w + 1, 2
        P = problem(nb, T, ns, nc, _seed("shape", case[1:]))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ins, out = run(P, dt, T, grad=True)
            torch.autograd.grad(out[2].sum(), [ins["Q"]])
            torch.cuda.synchronize()
        path = str(tmp_path / f"{_cid(case)}.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and "lqr_" in e.get("name", "")]
        names = sorted("bwd" if "lqr_bwd_kernel" in e["name"] else "fwd" for e in ev)
        assert names == ["bwd", "fwd"], (case, [e["name"] for e in ev])
        for e in ev:
            assert list(e["args"]["block"]) == [32 * w, 1, 1], (case, e["args"])
            assert list(e["args"]["grid"]) == [-(-nb // w), 1, 1], (case, e["args"])
