"""The linearisation, loss and predicted-reduction kernels of the pose-graph, two-pose and bundle-adjustment LM families
(csrc/lm.cu, ba.cu, pcg.cu, pcg2.cu) against the fp64 LM oracle, in fp32 and fp64, for robust kinds 0-6.

Tolerance, per output entry:  |got - ref| <= c * u * sum|term|
  ref        the fp64 oracle evaluated on the inputs after rounding them to the test dtype;
  u          the dtype's unit roundoff;
  sum|term|  the sum of the absolute values of the products that make the entry (oracle.lm_oracle *_terms companions:
             each factor enters with the magnitude of its own formula evaluated on absolute values, so translations
             computed with cancellation count with the size of the poses they come from, rotations composed from unit
             quaternions with O(1) entries);
  c          C_TERMS = 64 for every kernel and dtype.
The pose-graph reference uses lm_oracle.se3_Jl_inv_exact: the reference's closed forms of Jl^-1 and Q lose up to
~u / theta^4 to cancellation at small residual angles (1e-10 relative at theta ~ 1e-2 in fp64), far more than the kernels'
series, and would make the oracle, not the kernel, the larger error.
A missing, duplicated or sign-flipped row moves an entry by a whole term, far more than u * sum|term|; a bound relative to
the largest entry of an array would hide that in its small entries.  Scalars (losses, predicted reductions) use the same
rule with the sum|term| of their sum.  An entry whose sum|term| is 0 (an isolated node) must be exactly 0.

Sizes: every family runs a small problem and one past two rounds of the largest grid lm_grid launches (8 CTAs per SM):
per-thread kernels over > 2 * 8 * SMs * 128 items, the warp-per-pair kernels over > 2 * 8 * SMs * 4 pairs, the node-sum
and operator gathers over > 2 * 8 * SMs * 32 nodes, so the grid-stride loops run more than once and reduce_sums
(lm_common.cuh) folds more than 4 * 128 CTA partials in its unrolled loop.

Reproducibility: a second launch of every kernel without atomics gives bit-identical outputs and totals
(linearize_n, reproj2_accum_n, pgo2_node_sums, every loss, every predicted reduction, ba_linearize_seg,
ba_point_blocks, ba_wtx_gather).  lm_pgo_linearize / _w and lm_reproj2_accum (per-edge stores) are reproducible too and
the node-ordered stores are checked bit for bit against them.  lm_ba_linearize (stored rows) scatters Hcc / Hpp / gc / gp
with atomics and is exempt.
"""
import ctypes

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import lie_oracle as O
from oracle import lm_oracle as L
from tests.test_lm_gpu import _ba_geom, _ba_problem, cu

pytestmark = pytest.mark.gpu

C_TERMS = 64
UNIT = {torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
DTYPES = {"f32": torch.float32, "f64": torch.float64}
KINDS = range(7)
MEASURED = {}                   # largest |got - ref| / (u sum|term|) per (kernel output, dtype), over every case run
SENTINEL = 12345.0


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    """After the tests of this file that ran: the largest |got - ref| / (u sum|term|) of every kernel output and dtype."""
    MEASURED.clear()
    yield
    for k in sorted(MEASURED):
        print(f"\n{k:45s} {MEASURED[k]:8.3g}", end="")
    print()


def _np(t):
    return t.double().cpu().numpy()


class _Check:
    """Collects every bound violation of one test, so one failure shows all of them."""

    def __init__(self, dt):
        self.dt, self.u, self.fails = dt, UNIT[dt], []

    def __call__(self, name, got, ref, terms, c=C_TERMS):
        got = _np(got) if torch.is_tensor(got) else np.asarray(got, np.float64)
        ref, terms = np.asarray(ref, np.float64).reshape(got.shape), np.asarray(terms, np.float64).reshape(got.shape)
        err = np.abs(got - ref)
        assert np.isfinite(got).all(), name
        nz = terms > 0
        ratio = float((err[nz] / (self.u * terms[nz])).max()) if nz.any() else 0.0
        key = f"{name} {str(self.dt)[6:]}"
        MEASURED[key] = max(MEASURED.get(key, 0.0), ratio)
        if ratio > c or (err[~nz] != 0).any():
            self.fails.append(f"{name}: max |got-ref|/(u sum|term|) = {ratio:.3g} > {c}")

    def done(self):
        assert not self.fails, "\n".join(self.fails)


def _F():
    from pypose_b200.optim import _fused as F
    return F


def _ws_total(ws):
    return ws[:1].clone()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def _deltas(r):
    """delta of each robust kind: the median residual norm, so both branches of Huber occur."""
    d = float(np.median(np.sqrt((r ** 2).sum(-1))))
    return {k: (1.0 if k == 0 else (0.5 if k == 6 else d)) for k in KINDS}


# ------------------------------------------------------------------ pose graph
def _pgo_graph(rng, N, E_loop, hub):
    """Chain 0 .. N-2 (node N-1 isolated), random loop closures (both orders of i, j), a repeated edge, `hub` edges at node
    0; poses within a few units of the origin; measurements that leave residual rotations up to pi - 0.01."""
    nodes = O.exp("SE3", np.concatenate([rng.uniform(-1.5, 1.5, (N, 3)), rng.standard_normal((N, 3))], 1))
    ci, cj = rng.integers(0, N - 1, E_loop), rng.integers(0, N - 1, E_loop)
    hi, hj = np.zeros(hub, np.int64), rng.integers(1, N - 1, hub)
    ei = np.concatenate([np.arange(N - 2), ci, hi, hj[:hub // 2], [3, 3, 5]])
    ej = np.concatenate([np.arange(1, N - 1), cj, hj, hi[:hub // 2], [7, 7, 2]])
    keep = ei != ej
    ei, ej = ei[keep], ej[keep]
    E = len(ei)
    ang = np.where(rng.random(E) < 0.1, rng.uniform(0.0, np.pi - 0.01, E), np.abs(0.1 * rng.standard_normal(E)))
    ang[:2] = np.pi - 0.01
    ax = rng.standard_normal((E, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    xi = np.concatenate([0.1 * rng.standard_normal((E, 3)), ax * ang[:, None]], 1)
    Z = O.mul("SE3", O.mul("SE3", O.inv("SE3", nodes[ei]), nodes[ej]), O.exp("SE3", -xi))
    return nodes, Z, ei, ej


def _pgo_size(size):
    if size == "small":
        return 400, 300, 40
    return 2 * 8 * _sms() * 32 + 101, 2 * 8 * _sms() * 256, 4000


@pytest.mark.parametrize("size", ["small", "large"])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_pgo_linearize_paths(dtn, size):
    """lm_pgo_linearize, _n, _w (per-edge and shared W), lm_pgo_loss, pgo2_node_sums and the three predicted reductions."""
    F, dt = _F(), DTYPES[dtn]
    chk = _Check(dt)
    rng = np.random.default_rng(50 if size == "small" else 51)
    N, E_loop, hub = _pgo_size(size)
    nodes, Z, ei, ej = _pgo_graph(rng, N, E_loop, hub)
    E = len(ei)
    assert size == "small" or E >= 2 * 8 * _sms() * 256
    nd, Zd, eid, ejd = cu(nodes, dt), cu(Z, dt), _i32(ei), _i32(ej)
    nodes_r, Z_r = _np(nd), _np(Zd)
    r, J = L.pgo_jac_blocks(nodes_r, Z_r, ei, ej, exact=True)
    Jabs, rabs = L.pgo_terms(nodes_r, Z_r, ei, ej)
    assert np.abs(np.linalg.norm(r[:2, 3:], axis=1) - (np.pi - 0.01)).max() < 1e-4
    epos_i, epos_j, nptr, nother = L.node_layout(ei, ej, N)
    epi, epj, nptr_d, noth_d = _i32(epos_i), _i32(epos_j), _i32(nptr), _i32(nother)
    deltas = _deltas(r)
    ar = np.arange(E)
    Wb = rng.standard_normal((E, 6, 6))
    Wall = Wb @ np.swapaxes(Wb, -1, -2) / 6 + 0.5 * np.eye(6)
    ws = F._workspace(nd.device)
    for kind in KINDS:
        delta = deltas[kind]
        if kind == 1:
            nr = np.sqrt((r ** 2).sum(-1))
            assert (nr < delta).any() and (nr > delta).any()
        M_o, u_o, c_o = L.rows_linearize(J, r, ar, E, kind, delta)
        M_t, u_t, c_t = L.rows_terms(J, r, Jabs, rabs, ar, E, kind, delta)
        tag = f"pgo k{kind}"
        # per edge
        M, u = torch.empty(E, 21, dtype=dt, device="cuda"), torch.empty(E, 6, dtype=dt, device="cuda")
        F._launch("b200_lm_pgo_linearize", nd, [F._p(nd), F._p(Zd), F._p(eid), F._p(ejd), F._p(M), F._p(u), F._p(ws), kind,
                                                delta], E)
        cost = _ws_total(ws)
        chk("pgo_linearize M", M, M_o, M_t)
        chk("pgo_linearize u", u, u_o, u_t)
        chk("pgo_linearize cost", cost, c_o, c_t)
        # node order: the same blocks at both slots, -u at the first node's slot, padding untouched, same total
        Mn_runs = []
        for _ in range(2):
            Mn = torch.full((2 * E, 24), SENTINEL, dtype=dt, device="cuda")
            un = torch.full((2 * E, 6), SENTINEL, dtype=dt, device="cuda")
            F._launch("b200_lm_pgo_linearize_n", nd, [F._p(nd), F._p(Zd), F._p(eid), F._p(ejd), F._p(epi), F._p(epj), F._p(Mn),
                                                      F._p(un), F._p(ws), kind, delta], E)
            Mn_runs.append((Mn, un, _ws_total(ws)))
        Mn, un, cost_n = Mn_runs[0]
        assert all(torch.equal(a, b) for a, b in zip(Mn_runs[0], Mn_runs[1])), tag
        el, ejl = epi.long(), epj.long()
        assert torch.equal(Mn[el, :21], M) and torch.equal(Mn[ejl, :21], M), tag
        assert torch.equal(un[el], -u) and torch.equal(un[ejl], u), tag
        assert bool((Mn[:, 21:] == SENTINEL).all()), tag
        assert torch.equal(cost_n, cost), tag
        # node sums (atomic-free gather)
        sums = []
        for _ in range(2):
            Hd, g = torch.empty(N, 21, dtype=dt, device="cuda"), torch.empty(N, 6, dtype=dt, device="cuda")
            F._launch("b200_lm_pgo2_node_sums", nd, [F._p(Mn), F._p(un), F._p(nptr_d), F._p(Hd), F._p(g)], N)
            sums.append((Hd, g))
        Hd, g = sums[0]
        assert torch.equal(sums[1][0], Hd) and torch.equal(sums[1][1], g), tag
        Hd_o, g_o = L.pgo_scatter(M_o, u_o, ei, ej, N)
        Hd_t = L._group_sum(ei, M_t, N) + L._group_sum(ej, M_t, N)
        g_t = L._group_sum(ei, u_t, N) + L._group_sum(ej, u_t, N)
        chk("pgo2_node_sums Hd", Hd, Hd_o, Hd_t)
        chk("pgo2_node_sums g", g, g_o, g_t)
        assert not Hd[N - 1].any() and not g[N - 1].any()
        # loss
        losses = []
        for _ in range(2):
            F._launch("b200_lm_pgo_loss", nd, [F._p(nd), F._p(Zd), F._p(eid), F._p(ejd), F._p(ws), kind, delta], E)
            losses.append(_ws_total(ws))
        assert torch.equal(losses[0], losses[1]), tag
        chk("pgo_loss", losses[0], c_o, c_t)
        # information matrices: per edge and one shared (every kind on the small graph)
        for wname, Wc in ((("per-edge", Wall), ("shared", Wall[:1])) if size == "small" or kind < 2 else ()):
            Wd = cu(Wc.reshape(-1, 36), dt)
            W_r = np.broadcast_to(_np(Wd).reshape(-1, 6, 6), (E, 6, 6))
            outs = [torch.empty(E, w, dtype=dt, device="cuda") for w in (21, 6, 21, 6)]
            F._launch("b200_lm_pgo_linearize_w", nd, [F._p(nd), F._p(Zd), F._p(eid), F._p(ejd), F._p(Wd), 36 if len(Wc) > 1 else 0,
                                                      *[F._p(o) for o in outs], F._p(ws), kind, delta], E)
            Mw_o, uw_o, _ = L.rows_linearize(J, r, ar, E, kind, delta, W_r)
            Mw_t, uw_t, _ = L.rows_terms(J, r, Jabs, rabs, ar, E, kind, delta, W_r)
            chk(f"pgo_linearize_w M", outs[0], Mw_o, Mw_t)
            chk(f"pgo_linearize_w u", outs[1], uw_o, uw_t)
            chk(f"pgo_linearize_w M0", outs[2], M_o, M_t)
            chk(f"pgo_linearize_w u0", outs[3], u_o, u_t)
            chk(f"pgo_linearize_w cost", _ws_total(ws), c_o, c_t)
        if kind not in (0, 1):
            continue
        # predicted reductions at a random x, from the kernel's own blocks
        x = cu(rng.standard_normal((N, 6)), dt)
        xr, Mr, ur, gr = _np(x), _np(M), _np(u), _np(g)
        ref, terms = L.pgo_predicted(Mr, ur, ei, ej, xr, terms=True)
        terms += 2 * (np.abs(xr) * g_t).sum()          # the node sums g the two node-level kernels read carry their rounding
        for name, launch in (
                ("pgo_predicted", lambda: F._launch("b200_lm_pgo_predicted", M, [F._p(M), F._p(eid), F._p(ejd), E, F._p(x),
                                                                                  F._p(g), F._p(ws)], N)),
                ("pgo_predicted_edge", lambda: F._launch("b200_lm_pgo_predicted_edge", M, [F._p(M), F._p(u), F._p(eid), F._p(ejd),
                                                                                            F._p(x), F._p(ws)], E)),
                ("pgo2_predicted", lambda: F._launch("b200_lm_pgo2_predicted", M, [F._p(Mn), F._p(noth_d), F._p(nptr_d), F._p(x),
                                                                                    F._p(g), F._p(ws)], N))):
            got = []
            for _ in range(2):
                launch()
                got.append(_ws_total(ws))
            assert torch.equal(got[0], got[1]), name
            chk(name, got[0], [ref], [terms])
    chk.done()


# ------------------------------------------------------------------ two-pose reprojection
SKEW_K = (320.0, 0.7, 310.0, 300.0, 250.0)


def _reproj2_problem(rng, N, lengths, intr):
    """Pairs (a, b) with the given row counts, each followed by its reverse (b, a) when it has 31 rows or fewer; points
    in front of camera b, 10 % of them at the border of the image (|x / z| in [0.97, 1]); pixel noise with outliers."""
    fx = abs(intr[0])
    nodes = O.exp("SE3", np.concatenate([rng.uniform(-1.0, 1.0, (N, 3)), 0.5 * rng.standard_normal((N, 3))], 1))
    pa, pb, cnt = [], [], []
    for n in lengths:
        a = int(rng.integers(0, N))
        b = int((a + 1 + rng.integers(0, N - 1)) % N)
        pa.append(a); pb.append(b); cnt.append(n)
        if n <= 31:
            pa.append(b); pb.append(a); cnt.append(n)
    pa, pb, cnt = np.array(pa), np.array(pb), np.array(cnt)
    pseg = np.concatenate([[0], np.cumsum(cnt)])
    m = int(pseg[-1])
    pe = np.repeat(np.arange(len(pa)), cnt)
    ia, ib = pa[pe], pb[pe]
    z = rng.uniform(2.0, 6.0, m)
    xy = rng.uniform(-1.0, 1.0, (m, 2))
    border = rng.random(m) < 0.1
    xy[border, 0] = np.sign(xy[border, 0]) * rng.uniform(0.97, 1.0, border.sum())
    y = np.concatenate([xy * z[:, None], z[:, None]], 1)
    pts = O.act("SE3", O.mul("SE3", O.inv("SE3", nodes[ia]), nodes[ib]), y)
    fxy, sk, cx, fy, cy = intr
    proj = np.stack([(fxy * y[:, 0] + sk * y[:, 1]) / y[:, 2] + cx, fy * y[:, 1] / y[:, 2] + cy], 1)
    pix = proj + 0.01 * fx * rng.standard_normal((m, 2))
    out = rng.random(m) < 0.05
    pix[out] += 0.3 * fx * rng.standard_normal((out.sum(), 2))
    return nodes, pts, pix, pa, pb, pseg, ia, ib


@pytest.mark.parametrize("size", ["small", "large"])
@pytest.mark.parametrize("intr", ["readme", "skew"])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_reproj2_linearize_paths(dtn, intr, size):
    """lm_reproj2_accum, _accum_n, _loss, _residual, pgo2_node_sums and pgo2_predicted on pose pairs of 1, 31, 32, 33, 64
    and 10^4 rows (both orderings of the short ones) and, at the large size, > 2 * 8 * SMs * 4 pairs."""
    F, dt = _F(), DTYPES[dtn]
    chk = _Check(dt)
    K = L.README_INTR if intr == "readme" else SKEW_K
    rng = np.random.default_rng(60 if size == "small" else 61)
    lengths = [1, 31, 32, 33, 64, 10_000, 1, 2, 5]
    N = 40
    if size == "large":
        lengths += list(rng.integers(1, 7, 2 * 8 * _sms() * 4))
        N = 3000
    nodes, pts, pix, pa, pb, pseg, ia, ib = _reproj2_problem(rng, N, lengths, K)
    E, m = len(pa), int(pseg[-1])
    nd, td, xd = cu(nodes, dt), cu(pts, dt), cu(pix, dt)
    nodes_r, pts_r, pix_r = _np(nd), _np(td), _np(xd)
    pe = np.repeat(np.arange(E), np.diff(pseg))
    r, y = L.reproj2_residual(nodes_r, pts_r, pix_r, ia, ib, K)
    J = L.reproj2_jac_rows(nodes_r, pts_r, ia, ib, K)
    Jabs, rabs = L.reproj2_terms(nodes_r, pts_r, pix_r, ia, ib, K)
    ei, ej = pb, pa                                        # Reproj2Problem: J_b = -J, J_a = +J
    epos_i, epos_j, nptr, nother = L.node_layout(ei, ej, N)
    psd, pad, pbd, epi, epj, nptr_d, noth_d = (_i32(a) for a in (pseg, pa, pb, epos_i, epos_j, nptr, nother))
    kk = (ctypes.c_double * 5)(*K)
    ws = F._workspace(nd.device)
    # residual rows
    rd = torch.empty(m, 2, dtype=dt, device="cuda")
    iad, ibd = _i32(ia), _i32(ib)
    F._launch("b200_lm_reproj2_residual", nd, [F._p(nd), F._p(td), F._p(xd), F._p(iad), F._p(ibd), ctypes.addressof(kk), F._p(rd)], m)
    chk("reproj2_residual", rd, r, rabs)
    deltas = _deltas(r)
    for kind in KINDS:
        delta = deltas[kind]
        M_o, u_o, c_o = L.rows_linearize(J, r, pe, E, kind, delta)
        M_t, u_t, c_t = L.rows_terms(J, r, Jabs, rabs, pe, E, kind, delta)
        tag = f"reproj2 k{kind}"
        M, u = torch.empty(E, 21, dtype=dt, device="cuda"), torch.empty(E, 6, dtype=dt, device="cuda")
        F._launch("b200_lm_reproj2_accum", nd, [F._p(nd), F._p(td), F._p(xd), F._p(psd), F._p(pad), F._p(pbd), ctypes.addressof(kk),
                                                F._p(M), F._p(u), F._p(ws), kind, delta], E)
        cost = _ws_total(ws)
        chk("reproj2_accum M", M, M_o, M_t)
        chk("reproj2_accum u", u, u_o, u_t)
        chk("reproj2_accum cost", cost, c_o, c_t)
        runs = []
        for _ in range(2):
            Mn = torch.full((2 * E, 24), SENTINEL, dtype=dt, device="cuda")
            un = torch.full((2 * E, 6), SENTINEL, dtype=dt, device="cuda")
            F._launch("b200_lm_reproj2_accum_n", nd, [F._p(nd), F._p(td), F._p(xd), F._p(psd), F._p(pad), F._p(pbd),
                                                      ctypes.addressof(kk), F._p(epi), F._p(epj), F._p(Mn), F._p(un), F._p(ws),
                                                      kind, delta], E)
            runs.append((Mn, un, _ws_total(ws)))
        Mn, un, cost_n = runs[0]
        assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1])), tag
        el, ejl = epi.long(), epj.long()
        assert torch.equal(Mn[el, :21], M) and torch.equal(Mn[ejl, :21], M), tag
        assert torch.equal(un[el], -u) and torch.equal(un[ejl], u), tag
        assert bool((Mn[:, 21:] == SENTINEL).all()) and torch.equal(cost_n, cost), tag
        Hd, g = torch.empty(N, 21, dtype=dt, device="cuda"), torch.empty(N, 6, dtype=dt, device="cuda")
        F._launch("b200_lm_pgo2_node_sums", nd, [F._p(Mn), F._p(un), F._p(nptr_d), F._p(Hd), F._p(g)], N)
        Hd_o, g_o = L.pgo_scatter(M_o, u_o, ei, ej, N)
        Hd_t = L._group_sum(ei, M_t, N) + L._group_sum(ej, M_t, N)
        g_t = L._group_sum(ei, u_t, N) + L._group_sum(ej, u_t, N)
        chk("pgo2_node_sums(reproj2) Hd", Hd, Hd_o, Hd_t)
        chk("pgo2_node_sums(reproj2) g", g, g_o, g_t)
        losses = []
        for _ in range(2):
            F._launch("b200_lm_reproj2_loss", nd, [F._p(nd), F._p(td), F._p(xd), F._p(psd), F._p(pad), F._p(pbd),
                                                   ctypes.addressof(kk), F._p(ws), kind, delta], E)
            losses.append(_ws_total(ws))
        assert torch.equal(losses[0], losses[1]), tag
        chk("reproj2_loss", losses[0], c_o, c_t)
        if kind == 1:
            x = cu(rng.standard_normal((N, 6)), dt)
            ref, terms = L.pgo_predicted(_np(M), _np(u), ei, ej, _np(x), terms=True)
            terms += 2 * (np.abs(_np(x)) * g_t).sum()
            got = []
            for _ in range(2):
                F._launch("b200_lm_pgo2_predicted", M, [F._p(Mn), F._p(noth_d), F._p(nptr_d), F._p(x), F._p(g), F._p(ws)], N)
                got.append(_ws_total(ws))
            assert torch.equal(got[0], got[1])
            chk("pgo2_predicted(reproj2)", got[0], [ref], [terms])
    chk.done()


# ------------------------------------------------------------------ bundle adjustment
BA_LAYOUTS = [(1, 32), (1, 128), (3, 32), (2, 128)]


@pytest.mark.parametrize("size", ["small", "large"])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_ba_linearize_paths(dtn, size):
    """lm_ba_linearize (stored rows), ba_linearize_seg for every (split, tpi) layout of the PCG tests (small) or the one
    BAProblem picks (large, > 2 * 8 * SMs * 128 observations), ba_point_blocks, lm_ba_loss, ba_wtx_gather (with and
    without gp, alpha -1 and 1) and ba_predicted."""
    from pypose_b200.optim.structured import BAProblem
    F, dt = _F(), DTYPES[dtn]
    chk = _Check(dt)
    rng = np.random.default_rng(70 if size == "small" else 71)
    if size == "small":
        C, P = 12, 150
    else:
        C, P = 300, (2 * 8 * _sms() * 256) // 4 + 1000
    gt, ptsw, T0, p0, pix, cidx, pidx = _ba_problem(rng, C, P, 4, pix_noise=0.01, consecutive=True)
    out = rng.random(len(pix)) < 0.05
    pix[out] += 0.2 * rng.standard_normal((out.sum(), 2))
    o = np.argsort(cidx, kind="stable")
    pix, cidx, pidx = pix[o], cidx[o], pidx[o]
    m = len(cidx)
    Td, pd, xd = cu(T0, dt), cu(p0, dt), cu(pix, dt)
    T_r, p_r, pix_r = _np(Td), _np(pd), _np(xd)
    ci, pi_ = _i32(cidx), _i32(pidx)
    r = L.ba_residual(T_r, p_r, pix_r, cidx, pidx)
    y_o = O.act("SE3", T_r[cidx], p_r[pidx])
    Jc_abs, Jp_abs, rabs = L.ba_terms(T_r, p_r, pix_r, cidx, pidx)
    y_t = (np.abs(O.SO3_Adj(T_r[cidx][:, 3:])) @ np.abs(p_r[pidx])[..., None])[..., 0] + np.abs(T_r[cidx][:, :3])
    deltas = _deltas(r)
    if size == "small":
        layouts = BA_LAYOUTS
    else:
        prob = BAProblem(pp.module.BundleAdjustment(pp.SE3(Td), pd), xd, ci, pi_, None, None, (0, 1.0), 1e-4, 10)
        layouts = [tuple(prob.geom[1:3])]
    ws = F._workspace(Td.device)
    for kind in KINDS:
        delta = deltas[kind]
        outs_o = L.ba_linearize(T_r, p_r, pix_r, cidx, pidx, kind, delta)
        outs_t = L.ba_linearize_terms(T_r, p_r, pix_r, cidx, pidx, kind, delta)
        names = ("Jc", "Jp", "rs", "Hcc", "Hpp", "gc", "gp", "cost")
        # stored rows (atomics: not reproducible)
        outs = torch.ops.b200pose.lm_ba_linearize(Td, pd, xd, ci, pi_, kind, delta)
        for a, b, t, nm in zip(outs, outs_o, outs_t, names):
            chk(f"ba_linearize {nm}", a, b, t)
        # loss
        losses = []
        for _ in range(2):
            F._launch("b200_lm_ba_loss", Td, [F._p(Td), F._p(pd), F._p(xd), F._p(ci), F._p(pi_), F._p(ws), kind, delta], m)
            losses.append(_ws_total(ws))
        assert torch.equal(losses[0], losses[1])
        chk("ba_loss", losses[0], outs_o[7], outs_t[7])
        _, w = L.robust(kind, delta, (r ** 2).sum(-1))
        sw_t = np.sqrt(w * L._weight_factor(kind, delta, rabs))
        for split, tpi in layouts:
            geom, padj = _ba_geom(cidx, pidx, xd, C, P, split, tpi)
            padj_n = padj.cpu().numpy()
            runs = [F.ba_linearize_det(Td, pd, xd, pi_, geom, kind, delta) for _ in range(2)]
            (Y4, Y4p), rs, Hcc, Hpp, gc, gp, cur = runs[0]
            (Y4b, Y4pb), *rest = runs[1]
            assert torch.equal(Y4, Y4b) and torch.equal(Y4p, Y4pb), (kind, split, tpi)
            assert all(torch.equal(a, b) for a, b in zip((rs, Hcc, Hpp, gc, gp, cur), rest)), (kind, split, tpi)
            assert torch.equal(Y4p, Y4[padj]), (kind, split, tpi)
            lay = f"ba_linearize_seg {split}x{tpi}"
            chk(f"{lay} y", Y4[:, :3], y_o, y_t)
            chk(f"{lay} sqrt(w)", Y4[:, 3], np.sqrt(w), sw_t)
            chk(f"{lay} rs", rs, outs_o[2], outs_t[2])
            chk(f"{lay} Hcc", Hcc, outs_o[3], outs_t[3])
            chk(f"{lay} gc", gc, outs_o[5], outs_t[5])
            chk(f"{lay} cost", cur, outs_o[7], outs_t[7])
            chk("ba_point_blocks Hpp", Hpp, outs_o[4], outs_t[4])
            chk("ba_point_blocks gp", gp, outs_o[6], outs_t[6])
        # W^T x gather and the predicted reduction, from the deterministic route's rows (rebuilt from Y4 in the kernels)
        if kind not in (0, 1):
            continue
        cseg, split, tpi, ppos, cidx_p, pptr, pix_p = geom
        Y4r, Y4pr = _np(Y4), _np(Y4p)
        Jc_y, Jp_y = L.ba_rows_from_y(Y4r[:, :3], Y4r[:, 3], T_r, cidx)
        Jc_ya, Jp_ya = L.ba_rows_from_y(Y4r[:, :3], Y4r[:, 3], T_r, cidx, absolute=True)
        B = rng.standard_normal((P, 3, 3))
        iu3 = np.triu_indices(3)
        Hpinv = cu((np.eye(3) + B @ np.swapaxes(B, -1, -2) / 3)[:, iu3[0], iu3[1]], dt)
        hp = _np(Hpinv)
        Hpinv_r = np.zeros((P, 3, 3))
        Hpinv_r[:, iu3[0], iu3[1]] = hp
        Hpinv_r[:, iu3[1], iu3[0]] = hp
        x, xp = cu(rng.standard_normal((C, 6)), dt), cu(rng.standard_normal((P, 3)), dt)
        xr, xpr, gpr = _np(x), _np(xp), _np(gp)
        t_o = L.ba_wtx(Jc_y.reshape(-1, 12), Jp_y.reshape(-1, 6), cidx, pidx, xr, P)
        t_t = L.ba_wtx(Jc_ya.reshape(-1, 12), Jp_ya.reshape(-1, 6), cidx, pidx, np.abs(xr), P)
        for with_gp in (True, False):
            for alpha in (-1.0, 1.0):
                tt = t_o + (gpr if with_gp else 0.0)
                ta = t_t + (np.abs(gpr) if with_gp else 0.0)
                ref = alpha * (Hpinv_r @ tt[..., None])[..., 0]
                terms = (np.abs(Hpinv_r) @ ta[..., None])[..., 0]
                got = []
                for _ in range(2):
                    ud = torch.empty(P, 3, dtype=dt, device="cuda")
                    F._launch("b200_lm_ba_wtx_gather", Td, [F._p(Y4p), F._p(Td), F._p(cidx_p), F._p(pptr), F._p(Hpinv), F._p(x),
                                                            F._p(gp if with_gp else None), alpha, F._p(ud)], P)
                    got.append(ud)
                assert torch.equal(got[0], got[1])
                chk("ba_wtx_gather", got[0], ref, terms)
        ref = L.ba_predicted(Jc_y.reshape(-1, 12), Jp_y.reshape(-1, 6), _np(rs), cidx, pidx, xr, xpr)
        _, terms = L.ba_predicted(Jc_ya.reshape(-1, 12), Jp_ya.reshape(-1, 6), _np(rs), cidx, pidx, xr, xpr, terms=True)
        got = []
        for _ in range(2):
            F._launch("b200_lm_ba_predicted", Td, [F._p(Y4), F._p(Td), F._p(rs), F._p(ci), F._p(pi_), F._p(x), F._p(xp), F._p(ws)], m)
            got.append(_ws_total(ws))
        assert torch.equal(got[0], got[1])
        chk("ba_predicted", got[0], [ref], [terms])
    chk.done()
