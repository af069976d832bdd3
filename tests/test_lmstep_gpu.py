"""Device-decided LM trials (csrc/lmstep.cu) against fp64 oracles, in fp32 and fp64.

One C call runs a whole trial: linearise, accumulate, damped 6x6 solve, retraction and trial loss.  The last CTA then
decides (lm_decide) and lm_commit_kernel copies the trial poses into the parameters.  Every launch variant is called
through the ABI (`_lmstep.reproj_trial` / `poseinv_trial`) and compared with oracle/lm_oracle.py evaluated on the fp64
upcast of the kernel's inputs:

* H, g and the current loss per camera from the rows.  The damped solve (trial poses, predicted reduction, failed pivots)
  is the oracle's solve of the kernel's OWN H and g, so the accumulation and the solve are judged separately; the trial
  loss is the oracle's loss at the kernel's trial poses.
* Routes: register-fed with 8, 16 and 32 lanes per camera; TMA-staged; staged requested on a base one row off 16-byte
  alignment, which falls back to the register route and must be bit-identical to it.  Fresh trials and retries from the
  stored blocks, more cameras than one pass of the grid covers, failed pivots, and the decision and commit against the
  Python strategies bit for bit.

fp32 bounds, u = 2^-24 (fp64: the same formulas with u = 2^-53), per camera c of m_c rows:
  gamma_c   = 4 u (m_c / LPC + log2 LPC + 16)   (2 m_c / LPC sequential row adds per lane, the shuffle tree, and the
                                                 rounding of each row's terms; LPC = 32 for the staged kernel)
  H[c, ab]  <= gamma_c sum w |J_a|' |J_b|'   (|J|' = |J| + (|p| + |t| + |y|)(1 + |y|) / y_z^2, the terms of J)
  g[c, a]   <= gamma_c sum w |J_a|' s,        s = |r| + |pix| + |y| / y_z: the terms the residual is a difference of
  loss      <= sum_c gamma_c sum (rho terms + 2 w |r| s) + w (gamma_c s)^2   (rho terms: _rho_mag)
  D         <= 64 u kappa_c |D|_inf,   kappa_c = cond(damped block)
  trial pose <= (1 + |t|_inf) (bound on D + 16 u)
  predicted <= sum_c 64 u kappa_c (|D|^T |A| |D| + 2 |D|^T |g|)
The largest measured/bound ratio of each quantity is printed (run with -s) and recorded in DESIGN.md §4.
"""
import contextlib
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import lie_oracle as O
from oracle import lm_oracle as L
from tests.util import rand_group

ST_STATUS, ST_LOSS, ST_LAST, ST_DAMPING, ST_RADIUS, ST_DOWN, ST_REJECT, ST_CUR, ST_TRIAL, ST_PRED, ST_FAILED = range(11)
U = {torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
STAGES = {torch.float32: 4, torch.float64: 3}      # Staged<T>::kStages in lmstep.cu
TILE = 128                                           # Staged<T>::kRows
DMIN, DMAX = 1e-6, 1e32
IDS = {torch.float32: "f32", torch.float64: "f64"}

_worst = {}


def _within(key, err, bound):
    """err <= bound elementwise; keeps the largest err / bound per key for the printed summary."""
    err, bound = np.broadcast_arrays(np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64))
    assert np.isfinite(err).all(), key
    bad = err > bound
    assert not bad.any(), f"{key}: {bad.sum()} entries over the bound, worst err {err[bad].max():.3e} " \
                          f"bound {bound[bad][np.argmax(err[bad])]:.3e}"
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / bound, 0.0)
    _worst[key] = max(_worst.get(key, 0.0), float(r.max()) if r.size else 0.0)


def _report():
    print("\n" + "\n".join(f"  {k}: max err / bound = {v:.3g}" for k, v in sorted(_worst.items())))


def cu(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


def n64(t):
    return t.detach().double().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# oracle pieces
def _rho_mag(kind, delta, x):
    """Size of the terms rho(x) is computed from: several kernels subtract near-equal terms at small x (SoftLOne
    2 (delta sqrt(1/delta^2 + x) - 1), PseudoHuber, Huber's outer branch), so their rounding error is not relative to
    rho."""
    d2 = delta * delta
    with np.errstate(all="ignore"):
        if kind == 1:
            return np.where(np.sqrt(x) < delta, x, 2 * delta * np.sqrt(x) + d2)
        if kind == 2:
            return 2 * d2 * (np.sqrt(x / d2 + 1) + 1)
        if kind == 3:
            return d2 * (np.log(x / d2 + 1) + x / d2 + 1)
        if kind == 4:
            return 2 * (delta * np.sqrt(1 / d2 + x) + 1)
        if kind == 5:
            return d2 * (np.arctan(x / d2) + x / d2)
        if kind == 6:
            return abs(delta) * x
    return x


def _reproj_loss_terms(poses, pts, pix, seg, kind, delta):
    """Per camera: the loss, its bound magnitude sum (rho terms + 2 w |r| s) and sum w s^2 for the quadratic term."""
    C, m = poses.shape[0], int(seg[-1])
    cidx = np.repeat(np.arange(C), np.diff(seg))
    y = O.act("SE3", poses[cidx], pts[:m])
    r = -y[:, :2] / y[:, 2:] - pix[:m]
    x = (r ** 2).sum(-1)
    rho, w = L.robust(kind, delta, x)
    s = np.abs(r) + np.abs(pix[:m]) + (np.linalg.norm(y, axis=1) / y[:, 2])[:, None]
    return (L.seg_sum(rho, seg), L.seg_sum(_rho_mag(kind, delta, x) + 2 * w * (np.abs(r) * s).sum(1), seg),
            L.seg_sum(w * (s ** 2).sum(1), seg), s, w, cidx, y)


def _reproj_oracle(poses, pts, pix, seg, kind, delta):
    H, g, loss = L.reproj_accum_seg(poses, pts, pix, seg, kind, delta)
    _, lmag, lsq, s, w, cidx, y = _reproj_loss_terms(poses, pts, pix, seg, kind, delta)
    m = int(seg[-1])
    # |J| plus the size of the terms each entry is computed from: y = R p + t carries an error of u (|p| + |t|), which is
    # not small relative to a coordinate near 0 (x / z^2, x y / z^2, ... of J)
    ny, z = np.linalg.norm(y, axis=1), y[:, 2]
    e = (np.linalg.norm(pts[:m], axis=1) + np.linalg.norm(poses[cidx, :3], axis=1) + ny) / z
    aJ = np.abs(L.reproj_jac_rows(poses, pts[:m], cidx)) + (e * (1 + ny) / z)[:, None, None]
    iu = np.triu_indices(6)
    Hm = L.seg_sum(np.einsum('mka,mkb->mab', aJ, aJ)[:, iu[0], iu[1]] * w[:, None], seg)
    gm = L.seg_sum(np.einsum('mka,mk->ma', aJ, s) * w[:, None], seg)
    return dict(H=H, g=g, loss=loss, Hm=Hm, gm=gm, lmag=lmag, lsq=lsq)


def _solve_oracle(H21, g, poses, scale):
    """The oracle's damped solve and retraction of the given blocks, with the per-block condition number."""
    A = L._triu_unpack(H21)
    D, pred, failed = L.damped_solve_flagged(A, g, scale, DMIN, DMAX)
    idx = np.arange(6)
    Ad = A.copy()
    Ad[:, idx, idx] = np.clip(Ad[:, idx, idx], DMIN, DMAX) * scale
    kappa = np.linalg.cond(Ad)
    aD = np.abs(D)
    pmag = np.einsum('ci,cij,cj->c', aD, np.abs(A), aD) + 2 * (aD * np.abs(g)).sum(1)
    return dict(D=D, Pt=L.retract(D, poses), pred=pred, failed=failed, kappa=kappa, pmag=pmag)


def _gamma(u, m, lpc):
    return 4 * u * (m / lpc + math.log2(lpc) + 16)


def _loss_bound(gam, lmag, lsq):
    return float((gam * lmag + lsq * gam ** 2).sum())


# ---------------------------------------------------------------------------------------------------------------------
# harness: the ABI of the device-decided route, called the way optimizer.py calls it
class _Prob:
    """What _lmstep.reproj_trial / poseinv_trial read from a structured problem."""

    def __init__(self, poses, pts=None, pix=None, seg=None, X=None, robust=(0, 1.0)):
        self.poses, self.pts, self.pix, self.seg, self.X, self.robust = poses, pts, pix, seg, X, robust
        C = poses.shape[0]
        self._buf = (poses.new_empty(C, 21), poses.new_empty(C, 6), torch.empty_like(poses))
        self._trial = None

    def _poses(self):
        return self.poses

    def _rows(self):
        return self.poses, self.X


def _knobs():
    from pypose_b200 import _C
    lib = _C.lib()
    mode, lanes = lib.b200_lm_reproj_staged_mode, lib.b200_lm_reproj_lanes
    for f in (mode, lanes):
        f.restype, f.argtypes = ctypes.c_int, [ctypes.c_int]
    return mode, lanes


@contextlib.contextmanager
def _route(mode_v, lanes_v):
    """Both knobs are process-global: always restored."""
    mode, lanes = _knobs()
    prev_mode, prev_lanes = mode(-1), lanes(-1)
    try:
        mode(mode_v)
        lanes(lanes_v)
        yield
    finally:
        mode(prev_mode)
        lanes(prev_lanes)


def _fill(ds, strat, pg, last, cached, rc, limit):
    from pypose_b200.optim import _lmstep
    _lmstep.fill_ctl(ds.ctl, strat, pg, last, cached, rc, limit)


def _reject_ctl(ds, damping, rc):
    """Constant damping, a cached loss of -1 and a high reject limit: every trial is rejected, parameters stay put."""
    from pypose_b200.optim import strategy
    _fill(ds, strategy.Constant(damping), {'damping': damping}, -1.0, True, rc, 100)


def _call(ds, prob, scale, retry, poseinv=False, dmin=DMIN, dmax=DMAX):
    from pypose_b200.optim import _lmstep
    fn = _lmstep.poseinv_trial if poseinv else _lmstep.reproj_trial
    st_host = fn(ds, prob, scale, dmin, dmax, retry)
    torch.cuda.synchronize()
    st = ds.state.cpu().tolist()
    assert np.array_equal(st_host[:ST_FAILED + 1], st[:ST_FAILED + 1], equal_nan=True) and st_host[15] == float(ds.seq)
    Pt = prob._trial if poseinv else prob._buf[2]
    out = dict(st=st, Pt=Pt.clone(), poses=prob.poses.clone())
    if not poseinv:
        out["H"], out["g"] = prob._buf[0].clone(), prob._buf[1].clone()
    return out


def _same(a, b, keys):
    for k in keys:
        if k == "st":
            assert np.array_equal(a[k][:ST_FAILED + 1], b[k][:ST_FAILED + 1], equal_nan=True)
        else:
            assert torch.equal(a[k], b[k]), k


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# problems
def _problem(rng, counts, pix_noise=0.01, outliers=0.0, init_noise=0.1):
    counts = np.asarray(counts, np.int64)
    C, M = counts.size, int(counts.sum())
    cidx = np.repeat(np.arange(C), counts)
    gt = rand_group(rng, "SE3", C, tmax=0.5, t_sigma=0.5)
    pc = rng.uniform([-2, -2, 2], [2, 2, 6], (M, 3))
    pts = O.act("SE3", O.inv("SE3", gt)[cidx], pc)
    pix = -pc[:, :2] / pc[:, 2:] + pix_noise * rng.standard_normal((M, 2))
    bad = rng.random(M) < outliers
    pix[bad] += rng.uniform(-0.5, 0.5, (int(bad.sum()), 2))
    init = O.mul("SE3", O.exp("SE3", init_noise * rng.standard_normal((C, 6))), gt)
    seg = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    return init, pts, pix, seg


def _place(specs):
    """Row counts from (seg[c] % 4, count) specs: a filler camera of 1-3 rows goes before a list that has to start at a
    given offset from a 16-byte boundary."""
    counts, m = [], 0
    for mod, n in specs:
        if m % 4 != mod:
            counts.append((mod - m) % 4)
            m += counts[-1]
        counts.append(n)
        m += n
    return counts


def _ragged_counts(S):
    """0, 1, 3 rows; 4 LPC -+ 1 (the unrolled kAccRows loop and its remainder) for every width; 127 / 128 / 129 (one
    staged tile); e - floor(b/4)*4 = S*128 and S*128 + 1 (the last resident and the first streamed list of the ring);
    each with seg[c] % 4 = 0 and 3.  The last lists end inside the arrays' last, partial tile (copied by the lanes)."""
    span = S * TILE
    specs = []
    for mod in (0, 3):
        specs += [(mod, 0), (mod, 1), (mod, 3)]
        specs += [(mod, 4 * lpc + d) for lpc in (8, 16, 32) for d in (-1, 1)]
        specs += [(mod, n) for n in (127, 128, 129)]
        specs += [(mod, span - mod), (mod, span + 1 - mod), (mod, 2 * span + 5 - mod)]
    counts = _place(specs) + [1000, 0, 100, 2, 0]
    if sum(counts) % 4 == 0:
        counts[-2] += 1
    return counts


def _rounds_counts(rng, S, sms):
    """More cameras than one pass of the grid covers, for every route.  The staged kernel runs G = 8 SMs CTAs of 4 warps,
    one camera per warp, so cameras c, c + 4G, c + 8G, ... share a warp; by k = c // 4G they are resident (k % 4 = 0 or
    3), streamed (k % 4 = 1, in every eighth CTA) or empty (k % 4 = 2).  5 x 4G + 123 > 16 G cameras: the 8-lane kernel
    (16 cameras per CTA) runs two rounds, 16 lanes three, 32 lanes and staged six."""
    G = 8 * sms
    C = 5 * 4 * G + 123
    rd = np.arange(C) // 4
    k, cta = rd // G, rd % G
    counts = rng.integers(1, 41, C)
    big = rng.random(C) < 0.05
    counts[big] = rng.integers(41, S * TILE - 3, int(big.sum()))          # at most S tiles from any start
    streamed = (k % 4 == 1) & (cta % 8 == 0)
    counts[streamed] = S * TILE + 1 + rng.integers(0, 200, int(streamed.sum()))
    counts[k % 4 == 2] = 0
    return counts


def _staged_tiles(seg):
    b, e = seg[:-1].astype(np.int64), seg[1:].astype(np.int64)
    return np.where(e > b, (e - b // 4 * 4 + TILE - 1) // TILE, 0)


def _case(name, dt, rng):
    S = STAGES[dt]
    if name == "ragged":
        return _problem(rng, _ragged_counts(S), pix_noise=0.02, outliers=0.05)
    if name == "tiny":                                   # fewer rows than one tile in total
        return _problem(rng, [2, 0, 1, 3, 50, 0, 37, 5], pix_noise=0.02)
    if name == "mid":
        counts = rng.integers(0, 300, 301)
        counts[rng.random(301) < 0.05] = 0
        return _problem(rng, counts, pix_noise=0.05, outliers=0.05)
    if name == "rounds":
        counts = _rounds_counts(rng, S, _sms())
        init, pts, pix, seg = _problem(rng, counts, pix_noise=0.02, outliers=0.05)
        nt, G = _staged_tiles(seg), 8 * _sms()
        w0 = np.arange(0, 4 * 4 * G, 4 * G)              # the first four cameras of warp 0 of CTA 0
        assert nt[w0[0]] <= S and nt[w0[1]] > S and nt[w0[2]] == 0 and 0 < nt[w0[3]] <= S
        return init, pts, pix, seg
    raise KeyError(name)


# route name, staged mode, lanes knob, LPC of the bounds (None: the default width), one row off 16-byte alignment
ROUTES = [("reg8", 0, 8, 8, False), ("reg16", 0, 16, 16, False), ("reg32", 0, 32, 32, False), ("staged", 2, 0, 32, False),
          ("staged-misaligned", 2, 0, None, True)]


def _offset(t):
    """The same rows on a base one row past a 16-byte boundary."""
    buf = torch.empty((t.shape[0] + 1,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    v = buf[1:]
    v.copy_(t)
    return v


def _check_trial(tag, out, orc, P64, X64, Z64, seg, kind, delta, scale, gam, u, retry):
    """One trial against the oracle: blocks (fresh only), solve of the kernel's blocks, the four sums, the state."""
    st = out["st"]
    H, g, Pt = n64(out["H"]), n64(out["g"]), n64(out["Pt"])
    if not retry:
        _within(f"{tag} H", np.abs(H - orc["H"]), gam[:, None] * orc["Hm"])
        _within(f"{tag} g", np.abs(g - orc["g"]), gam[:, None] * orc["gm"])
        _within(f"{tag} cur loss", abs(st[ST_CUR] - orc["loss"].sum()), _loss_bound(gam, orc["lmag"], orc["lsq"]))
    else:
        assert st[ST_CUR] == 0.0          # a retry does not reread the rows; the host uses ST_CUR of the first trial only
    so = _solve_oracle(H, g, P64, scale)
    assert st[ST_FAILED] == float(so["failed"].sum())
    ok = ~so["failed"]
    dbound = 64 * u * so["kappa"] * np.abs(so["D"]).max(1)
    tmax = np.abs(P64[:, :3]).max(1)
    _within(f"{tag} trial pose", np.abs(Pt - so["Pt"]).max(1)[ok], ((1 + tmax) * (dbound + 16 * u))[ok])
    _within(f"{tag} predicted", abs(st[ST_PRED] - so["pred"].sum()), (64 * u * so["kappa"] * so["pmag"])[ok].sum())
    tl, tmag, tsq = _reproj_loss_terms(Pt, X64, Z64, seg, kind, delta)[:3]
    _within(f"{tag} trial loss", abs(st[ST_TRIAL] - tl.sum()), _loss_bound(gam, tmag, tsq))
    # the control block: Constant, cached loss -1 -> rejected, parameters untouched
    assert st[ST_STATUS] == 0.0 and st[ST_LOSS] == -1.0 and st[ST_LAST] == -1.0
    assert st[ST_REJECT] == (2.0 if retry else 1.0)
    assert torch.equal(out["poses"], out["P0"])


CASES = [("ragged", 0, 1.0), ("ragged", 1, 0.05), ("tiny", 0, 1.0)] + \
        [("mid", k, d) for k, d in ((1, 0.05), (2, 0.05), (3, 0.1), (4, 0.1), (5, 0.3), (6, 0.5))] + \
        [("rounds", 0, 1.0), ("rounds", 1, 0.05)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,kind,delta", CASES, ids=[f"{c}-k{k}" for c, k, _ in CASES])
@pytest.mark.parametrize("dt", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_reproj_trial_every_route_vs_fp64_oracle(dt, case, kind, delta):
    """Every route of b200_lm_reproj_step, fresh and retried, against the per-camera fp64 oracle; each call run twice is
    bit-identical (no float atomics), the misaligned base falls back to the register route bit for bit."""
    from pypose_b200.optim import _lmstep
    rng = np.random.default_rng(zlib.crc32(f"{case}-{kind}".encode()))
    init, pts, pix, seg = _case(case, dt, rng)
    P, X, Z, segd = cu(init, dt), cu(pts, dt), cu(pix, dt), torch.from_numpy(seg).cuda()
    P64, X64, Z64 = n64(P), n64(X), n64(Z)
    orc = _reproj_oracle(P64, X64, Z64, seg, kind, delta)
    m = np.diff(seg).astype(np.float64)
    u = U[dt]
    scale1, scale2 = 1.0 + 1e-2, (1.0 + 1e-2) * (1.0 + 0.5)
    C, M = P.shape[0], X.shape[0]
    for name, mode, lanes, lpc, misaligned in ROUTES:
        if lpc is None:
            lpc = 32 if M >= 384 * C else 8
        tag = f"{IDS[dt]} {name}"
        Xd, Zd = (_offset(X), _offset(Z)) if misaligned else (X, Z)
        if misaligned:
            assert Xd.data_ptr() % 16 != 0
        prob = _Prob(P.clone(), Xd, Zd, segd, robust=(kind, delta))
        ds = _lmstep.DeviceStep(P.device, dt)
        ds.new_state()
        P0 = prob.poses.clone()
        with _route(mode, lanes):
            _reject_ctl(ds, 1e-2, 0)
            a = _call(ds, prob, scale1, False)
            b = _call(ds, prob, scale1, False)
            _same(a, b, ("H", "g", "Pt", "st"))
            _reject_ctl(ds, 0.5, 1)
            r = _call(ds, prob, scale2, True)
            assert torch.equal(r["H"], a["H"]) and torch.equal(r["g"], a["g"])      # a retry leaves the blocks alone
        if misaligned:
            with _route(0, 0):
                _reject_ctl(ds, 1e-2, 0)
                ref = _call(ds, prob, scale1, False)
                _reject_ctl(ds, 0.5, 1)
                ref_r = _call(ds, prob, scale2, True)
            _same(a, ref, ("H", "g", "Pt", "st"))
            _same(r, ref_r, ("Pt", "st"))
        gam = _gamma(u, m, lpc)
        for out, retry, scale in ((a, False, scale1), (r, True, scale2)):
            out["P0"] = P0
            _check_trial(tag, out, orc, P64, X64, Z64, seg, kind, delta, scale, gam, u, retry)
    _report()


def _indefinite_packed():
    A = np.eye(6)
    A[0, 1] = A[1, 0] = 1e8                          # indefinite under any damping scale a test uses
    return L._triu_pack(A)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_reproj_retry_on_indefinite_blocks_fails_and_keeps_parameters(dt):
    """A retry on stored blocks of which k are indefinite: ST_FAILED = k, status 2, the loss stays the cached one and the
    parameters are bit for bit unchanged, on every route; the other cameras' trial poses still solve their blocks."""
    from pypose_b200.optim import _lmstep, strategy
    rng = np.random.default_rng(21)
    init, pts, pix, seg = _case("ragged", dt, rng)
    P, X, Z, segd = cu(init, dt), cu(pts, dt), cu(pix, dt), torch.from_numpy(seg).cuda()
    C, counts = P.shape[0], np.diff(seg)
    bad = np.array([np.flatnonzero(counts == 0)[0], np.flatnonzero(counts == 1)[0], C // 2, C - 1])
    assert counts[bad[-1]] == 0                      # an empty camera, a 1-row camera, one in the middle, the last
    u = U[dt]
    for name, mode, lanes, _, _ in ROUTES[:4]:
        prob = _Prob(P.clone(), X, Z, segd)
        ds = _lmstep.DeviceStep(P.device, dt)
        ds.new_state()
        with _route(mode, lanes):
            _reject_ctl(ds, 1e-2, 0)
            _call(ds, prob, 1.01, False)
            prob._buf[0][torch.from_numpy(bad).cuda()] = cu(_indefinite_packed(), dt)
            P0 = prob.poses.clone()
            # a cached loss no trial can miss: without the failed pivots this trial would be accepted and committed
            _fill(ds, strategy.TrustRegion(), dict(strategy.TrustRegion().defaults), 1e30, True, 1, 16)
            out = _call(ds, prob, 1.5, True)
        st = out["st"]
        assert st[ST_FAILED] == float(len(bad)) and st[ST_STATUS] == 2.0, (name, st)
        assert st[ST_LOSS] == 1e30 and st[ST_REJECT] == 1.0 and st[ST_DAMPING] == 1e-6
        assert torch.equal(out["poses"], P0), name
        so = _solve_oracle(n64(out["H"]), n64(out["g"]), n64(P0), 1.5)
        assert so["failed"][bad].all() and so["failed"].sum() == len(bad)
        ok = ~so["failed"]
        bound = (1 + np.abs(n64(P0)[:, :3]).max(1)) * (64 * u * so["kappa"] * np.abs(so["D"]).max(1) + 16 * u)
        _within(f"{IDS[dt]} {name} trial pose beside failed blocks", np.abs(n64(out["Pt"]) - so["Pt"]).max(1)[ok], bound[ok])


# ---------------------------------------------------------------------------------------------------------------------
# PoseInv
POSEINV_KINDS = [(0, 1.0), (1, 0.05), (2, 0.05), (3, 0.1), (4, 0.1), (5, 0.3), (6, 0.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,delta", POSEINV_KINDS, ids=[f"k{k}" for k, _ in POSEINV_KINDS])
@pytest.mark.parametrize("dt", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_poseinv_trial_vs_fp64_oracle(dt, kind, delta):
    """b200_lm_poseinv_step per pose and in the four sums, from one pose to more than 8 SMs x 128 (the grid-stride
    loop).  Per pose i, s_i = 1 + |t_P| + |t_X| (the size of the terms of Log(P X)); kappa_i of the damped block:
      trial pose <= 64 u kappa_i s_i (1 + |D_i|) (1 + |t_P|);  sums: 64 u (rho terms + 2 w |r| s) + w (64 u s)^2 summed,
      predicted: 64 u kappa_i s_i (|D|^T |A| |D| + 2 |D|^T |g|) summed."""
    from pypose_b200.optim import _lmstep
    rng = np.random.default_rng(7 + kind)
    n_max = 8 * _sms() * 128 + 4099
    Pall, Xall = rand_group(rng, "SE3", n_max, tmax=2.0), rand_group(rng, "SE3", n_max, tmax=2.0)
    u, scale = U[dt], 1.0001
    gam = 64 * u
    for n in (1, 127, 20011, n_max):
        P, X = cu(Pall[:n], dt), cu(Xall[:n], dt)
        P64, X64 = n64(P), n64(X)
        prob = _Prob(P.clone(), X=X, robust=(kind, delta))
        ds = _lmstep.DeviceStep(P.device, dt)
        ds.new_state()
        _reject_ctl(ds, 1e-4, 0)
        out = _call(ds, prob, scale, False, poseinv=True)
        st = out["st"]
        assert torch.equal(out["poses"], P) and st[ST_STATUS] == 0.0 and st[ST_FAILED] == 0.0
        r, J = L.poseinv_jac_blocks(P64, X64)
        rho, w = L.robust(kind, delta, (r ** 2).sum(-1))
        A = np.swapaxes(J, -1, -2) @ J * w[:, None, None]
        gv = (np.swapaxes(J, -1, -2) @ r[..., None])[..., 0] * w[:, None]
        so = _solve_oracle(L._triu_pack(A), gv, P64, scale)
        assert not so["failed"].any()
        s = 1 + np.abs(P64[:, :3]).max(1) + np.abs(X64[:, :3]).max(1)
        tP = np.abs(P64[:, :3]).max(1)
        tag = f"{IDS[dt]} poseinv"
        _within(f"{tag} trial pose", np.abs(n64(out["Pt"]) - so["Pt"]).max(1),
                gam * so["kappa"] * s * (1 + np.abs(so["D"]).max(1)) * (1 + tP))
        rn = np.linalg.norm(r, axis=1)
        rm = _rho_mag(kind, delta, rn ** 2)
        _within(f"{tag} cur loss", abs(st[ST_CUR] - rho.sum()), (gam * (rm + 2 * w * rn * s) + w * (gam * s) ** 2).sum())
        _within(f"{tag} predicted", abs(st[ST_PRED] - so["pred"].sum()), (gam * so["kappa"] * s * so["pmag"]).sum())
        rt = L.poseinv_residual(n64(out["Pt"]), X64)
        rho_t, w_t = L.robust(kind, delta, (rt ** 2).sum(-1))
        rtn = np.linalg.norm(rt, axis=1)
        _within(f"{tag} trial loss", abs(st[ST_TRIAL] - rho_t.sum()),
                (gam * (_rho_mag(kind, delta, rtn ** 2) + 2 * w_t * rtn * s) + w_t * (gam * s) ** 2).sum())
    _report()


# ---------------------------------------------------------------------------------------------------------------------
# the decision and the commit on the device
def _random_strategy(rng, kind):
    from pypose_b200.optim import strategy
    if kind == 0:
        return strategy.Constant(damping=float(10 ** rng.uniform(-6, 0)))
    if kind == 1:
        return strategy.Adaptive(damping=float(10 ** rng.uniform(-6, 0)), high=0.5, low=1e-3, up=float(rng.uniform(1.5, 4)),
                                 down=float(rng.uniform(0.1, 0.9)))
    return strategy.TrustRegion(radius=float(10 ** rng.uniform(0, 6)), up=float(rng.uniform(1.5, 4)),
                                down=float(rng.uniform(0.1, 0.9)), factor=float(rng.uniform(0.1, 0.9)))


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["register", "staged", "poseinv"])
@pytest.mark.parametrize("dt", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_device_decision_and_commit_equal_python_strategies(dt, family):
    """~200 random control blocks per deciding kernel (fill_ctl over the three strategies, cached or not, reject counts
    below, at and above the limit, fresh trials, retries and retries on failed pivots).  The device state equals
    strategy.update plus the accept rule of optimizer.py applied to the (cur, trial, predicted, failed) it reports, bit
    for bit; the pinned host copy equals it with the sequence number in slot 15; status 1 commits the trial poses bit for
    bit, status 0 and 2 leave the parameters bit for bit unchanged."""
    from pypose_b200.optim import _lmstep
    rng = np.random.default_rng({"register": 31, "staged": 32, "poseinv": 33}[family])
    poseinv = family == "poseinv"
    if poseinv:
        n = 500
        prob = _Prob(cu(rand_group(rng, "SE3", n, tmax=2.0), dt), X=cu(rand_group(rng, "SE3", n, tmax=2.0), dt))
        knobs = (0, 0)
    else:
        init, pts, pix, seg = _problem(rng, rng.integers(10, 300, 40), pix_noise=0.03, init_noise=0.2)
        prob = _Prob(cu(init, dt), cu(pts, dt), cu(pix, dt), torch.from_numpy(seg).cuda())
        knobs = (2, 0) if family == "staged" else (0, 8)
    ds = _lmstep.DeviceStep(prob.poses.device, dt)
    ds.new_state()
    seen = {0.0: 0, 1.0: 0, 2.0: 0}
    with _route(*knobs):
        _reject_ctl(ds, 1e-2, 0)
        cur_ref = _call(ds, prob, 1.01, False, poseinv)["st"][ST_CUR]
        poisoned, have_blocks = 0, True
        for i in range(200):
            kind = i % 3
            strat = _random_strategy(rng, kind)
            pg = dict(strat.defaults)
            pg['damping'] = float(10 ** rng.uniform(-6, 2))
            if kind == 2:
                pg['down'] = float(10 ** rng.uniform(-5, 0))
            last = cur_ref if rng.random() < 0.1 else float(cur_ref * 10 ** rng.uniform(-0.5, 0.3))
            cached = bool(rng.random() < 0.7)
            rc, limit = int(rng.integers(0, 4)), int(rng.integers(0, 4))
            retry = have_blocks and rng.random() < 0.3
            if retry and rng.random() < 0.2:
                if poseinv:                                # a negative diagonal clamp fails the first pivot of every pose
                    poisoned = n
                else:
                    k = int(rng.integers(1, 4))
                    prob._buf[0][:k] = cu(_indefinite_packed(), dt)
                    poisoned = k
            elif not retry:
                poisoned = 0
            scale = (1.0 + pg['damping']) * (float(rng.uniform(1.5, 3)) if retry else 1.0)
            _fill(ds, strat, pg, last, cached, rc, limit)
            P0 = prob.poses.clone()
            clamp = (-2.0, -1.0) if poseinv and poisoned else (DMIN, DMAX)
            out = _call(ds, prob, scale, retry, poseinv, *clamp)
            st = out["st"]
            cur, trial, pred, failed = st[ST_CUR:ST_FAILED + 1]
            # PoseInv has no stored blocks: its retry relinearises and reports the current loss
            if retry and not poseinv:
                assert cur == 0.0
            elif not failed:
                cur_ref = cur
            assert failed == float(poisoned), (i, failed, poisoned)
            if poseinv:
                poisoned = 0
            eff_last = last if cached else cur
            assert st[ST_LAST] == eff_last
            seen[st[ST_STATUS]] += 1
            if failed:
                assert st[ST_STATUS] == 2.0 and st[ST_LOSS] == eff_last and st[ST_REJECT] == rc
                assert st[ST_DAMPING] == pg['damping'] and torch.equal(out["poses"], P0)
                continue
            ref_pg = dict(pg)
            strat.update(ref_pg, last=eff_last, loss=trial, J=None, D=None, R=None, predicted=pred)
            reject = eff_last < trial and rc < limit
            assert st[ST_STATUS] == (0.0 if reject else 1.0), i
            assert st[ST_LOSS] == (eff_last if reject else trial)
            assert st[ST_REJECT] == (rc + 1 if reject else rc)
            got = dict(pg)
            _lmstep.apply_state(strat, got, st)
            assert got == ref_pg, (i, kind, got, ref_pg)
            if reject:
                assert torch.equal(out["poses"], P0), i
            else:
                assert torch.equal(out["poses"], out["Pt"]), i
    assert min(seen.values()) >= 3, seen


# ---------------------------------------------------------------------------------------------------------------------
# end to end: device-decided route against the host-decided route
@pytest.mark.gpu
def test_lm_steps_device_route_equal_host_route_without_device_step(monkeypatch):
    """2e4 cameras, 5 % gross outliers, Huber, TrustRegion from a poor start, so that the trust region shrinks through
    rejected trials within six LM.steps.  The device-decided route and the host-decided route (lm.cu kernels, decision
    in Python) give the same reject counts, losses to 1e-9 relative and poses to 1e-8 in fp64.  Cameras whose rows are
    mostly down-weighted outliers have blocks with condition numbers up to ~1e9 here, which the two summation orders
    turn into differences of a few 1e-10 after six steps.  fp32 is not compared end to end: at u kappa > 1 the two fp32
    trajectories part on such cameras from the first step, while every fp32 trial is pinned per camera above."""
    import pypose_b200 as pp
    from pypose_b200.optim import structured
    dt, ltol, ptol = torch.float64, 1e-9, 1e-8
    rng = np.random.default_rng(41)
    counts = rng.integers(5, 46, 20000)
    init, pts, pix, seg = _problem(rng, counts, pix_noise=0.01, outliers=0.05, init_noise=0.25)
    cidx = np.repeat(np.arange(counts.size), counts)
    inp = (cu(pts, dt), cu(pix, dt), torch.from_numpy(cidx).cuda())
    runs = {}
    for host in (False, True):
        if host:
            monkeypatch.setattr(structured.ReprojProblem, "device_step", lambda self, strategy: None)
        net = pp.module.PoseReproj(pp.SE3(cu(init, dt)))
        opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(radius=1e6), kernel=pp.optim.kernel.Huber(delta=0.05))
        losses, rejects = [], []
        for _ in range(6):
            losses.append(float(opt.step(inp)))
            rejects.append(opt.reject_count)
        assert (getattr(opt._problem, "_ds", None) is None) == host
        runs[host] = (np.array(losses), rejects, n64(net.poses))
    print(f"\n  losses {runs[False][0]} rejects {runs[False][1]}; host route {runs[True][0]} {runs[True][1]}")
    print(f"  max |loss rel diff| {np.abs(runs[False][0] / runs[True][0] - 1).max():.3e}, "
          f"max |pose diff| {np.abs(runs[False][2] - runs[True][2]).max():.3e}")
    assert sum(runs[False][1]) > 0
    assert runs[False][1] == runs[True][1]
    np.testing.assert_allclose(runs[False][0], runs[True][0], rtol=ltol)
    assert np.abs(runs[False][2] - runs[True][2]).max() <= ptol


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's segment reduction (CPU)
def test_segment_reduction_oracle_equals_add_at():
    """lm_oracle.reproj_accum_seg (np.add.reduceat over camera-sorted rows, empty cameras included) against
    reproj_accum (np.add.at), and damped_solve_flagged against damped_solve on the blocks it does not flag."""
    rng = np.random.default_rng(0)
    counts = [0, 3, 1, 0, 17, 2, 0, 40, 0]
    init, pts, pix, seg = _problem(rng, counts, pix_noise=0.05)
    empty = np.diff(seg) == 0
    for kind, delta in ((0, 1.0), (1, 0.05), (3, 0.1)):
        H, g, loss = L.reproj_accum_seg(init, pts, pix, seg, kind, delta)
        H_o, g_o, s_o = L.reproj_accum(init, pts, pix, seg, kind, delta)
        assert np.abs(H - H_o).max() <= 1e-13 * np.abs(H_o).max()
        assert np.abs(g - g_o).max() <= 1e-13 * np.abs(g_o).max()
        np.testing.assert_allclose(loss.sum(), s_o[0], rtol=1e-13)
        assert (H[empty] == 0).all() and (g[empty] == 0).all() and (loss[empty] == 0).all()
    A = L._triu_unpack(H_o)
    A[[1, 4]] = L._triu_unpack(_indefinite_packed())
    D, pred, failed = L.damped_solve_flagged(A, g_o, 1.5, DMIN, DMAX)
    assert failed.tolist() == [c in (1, 4) for c in range(len(counts))]
    D_o, pred_o = L.damped_solve(A[~failed], g_o[~failed], 1.5, DMIN, DMAX)
    assert np.array_equal(D[~failed], D_o) and np.array_equal(pred[~failed], pred_o)
    assert (D[failed] == 0).all() and (pred[failed] == 0).all()
    with pytest.raises(np.linalg.LinAlgError):
        L.damped_solve(A, g_o, 1.5, DMIN, DMAX)
