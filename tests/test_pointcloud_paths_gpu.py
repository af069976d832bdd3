"""Every launch path of csrc/knn.cu against fp64 oracles (oracle/icp_oracle.py, oracle/pcfilter_oracle.py, scipy's
cKDTree), in fp32 and fp64.  Which kernel runs is chosen at run time from the shapes and the SM count (DESIGN.md §3.4,
§3.5); every test asserts the path it reached, so that a change of the planning rules cannot move a case off its path:

* k-NN: split or not from `b200_knn_workspace_bytes` (> 0 when the N2 range is split), with the plan mirrored here;
* ICP: the source points per CTA from `b200_icp_workspace_bytes(B, Ns) = (16 + 12 B + 17 B nx) 8`;
* radius mask: four queries per thread when ceil(N / 1024) >= 2 SMs.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import icp_oracle as O
from oracle import pcfilter_oracle as PF

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
ORDS = (1, 2, math.inf)
K_EDGES = (1, 2, 4, 5, 8, 9, 16, 17, 32)          # both ends of the buckets 1, 4, 8, 16, 32
GENERAL_D = (1, 2, 4, 7, 16, 1, 2, 4, 7)           # D != 3, paired with K_EDGES


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lib_fn(name, nargs):
    from pypose_b200 import _C
    f = getattr(_C.lib(), name)
    f.restype, f.argtypes = ctypes.c_longlong, [ctypes.c_longlong] * nargs
    return f


def _kbucket(k):
    return 1 if k <= 1 else 4 if k <= 4 else 8 if k <= 8 else 16 if k <= 16 else 32


def _knn_plan(B, N1, N2, D, k):
    """knn_plan of csrc/knn.cu -> (query blocks, splits S, chunk, K bucket); checked against the library below."""
    K = _kbucket(k)
    Q = 1 if D != 3 else 4 if K == 1 else 2 if K == 4 else 1
    nqb = -(-N1 // (256 * Q))
    base, want = B * nqb, 4 * _sms()
    S = 1
    if 0 < base < want:
        S = max(1, min(-(-want // base), -(-N2 // 2048), 64))
    chunk = max(-(-(-(-N2 // S)) // 256) * 256, 256)
    return nqb, -(-N2 // chunk), chunk, K


def knn_path(B, N1, N2, D, k, dt):
    """-> (split?, chunk): the workspace size the library asks for must be the one of the mirrored plan."""
    elem = 4 if dt == F32 else 8
    with torch.cuda.device(0):
        ws = int(_lib_fn("b200_knn_workspace_bytes", 6)(B, N1, N2, D, k, elem))
    _, S, chunk, K = _knn_plan(B, N1, N2, D, k)
    n = S * B * N1 * K
    assert ws == (0 if S == 1 else -(-n * elem // 256) * 256 + 4 * n), (B, N1, N2, D, k, ws)
    return S > 1, chunk


def icp_nx(B, Ns):
    with torch.cuda.device(0):
        ws = int(_lib_fn("b200_icp_workspace_bytes", 2)(B, Ns))
    nx, rem = divmod(ws // 8 - 16 - 12 * B, 17 * B)
    assert rem == 0 and ws % 8 == 0
    return nx


def _rows(N1, n=40):
    """A query subsample: an even spread plus both sides of every 256-query block edge and the last queries."""
    edges = [e + o for e in range(256, N1, 256) for o in (-1, 0)]
    return np.unique(np.clip(np.r_[np.linspace(0, N1 - 1, n).astype(int), edges, N1 - 2, N1 - 1], 0, N1 - 1))


def _randn(shape, seed, dt, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, dtype=F64, generator=g) * scale).to(dt)


def check_knn(v, i, rq, nb, k, ordv, largest, dt, what=""):
    """v, i (M, k) from the kernel for the queries rq (M, D) against nb (N2, D), both the fp64 upcast of its inputs.
    fp64: the oracle's indices exactly and values to 1e-13.  fp32: values to 1e-6, and indices equal wherever the fp64
    distances of neighbouring ranks differ by more than 1e-5 relative."""
    rv, ri = O.knn(rq, nb, k, ordv, largest)
    assert i.shape == ri.shape, what
    if dt == F64:
        np.testing.assert_array_equal(i, ri, err_msg=what)
        np.testing.assert_allclose(v, rv, rtol=1e-13, atol=1e-14, err_msg=what)
        return
    np.testing.assert_allclose(v, rv, rtol=1e-6, atol=1e-6, err_msg=what)
    d = O.distances(rq, nb, ordv)
    np.testing.assert_allclose(np.take_along_axis(d, i, -1), rv, rtol=2e-6, atol=2e-6, err_msg=what)
    full = np.sort(-d if largest else d, -1)
    pad = np.full(full.shape[:-1] + (1,), np.inf)
    ext = np.concatenate([-pad, full, pad], -1)
    thr = 1e-5 * (1 + np.abs(full[..., :k]))
    clear = (ext[..., 1:k + 1] - ext[..., :k] > thr) & (ext[..., 2:k + 2] - ext[..., 1:k + 1] > thr)
    assert (i[clear] == ri[clear]).all(), what


def _np(t):
    return t.detach().double().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# k-NN
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F32, F64])
@pytest.mark.parametrize("ordv", ORDS)
def test_knn_every_instantiation_vs_oracle(dt, ordv):
    """Every (D class, K bucket, largest, split) of knn_kernel / knn_merge_kernel for this dtype and ord, at k on both
    edges of every bucket, D in {1, 2, 3, 4, 7, 16} and N1 = 777 (not a multiple of 256 Q: the last thread's extra
    queries of Q = 2 and Q = 4 are clamped).  Split: B = 1, N2 = 9000.  Unsplit: N2 = 3000 and a batch of
    ceil(4 SMs / query blocks) elements; the first and last element are compared."""
    N1, n2_split, n2_whole = 777, 9000, 3000
    reached = set()
    rows = _rows(N1)
    data = {}
    for D, k in [(3, k) for k in K_EDGES] + list(zip(GENERAL_D, K_EDGES)):
        nqb, _, _, K = _knn_plan(1, N1, n2_split, D, k)
        B = -(-4 * _sms() // nqb)
        for split, Bc, N2 in ((True, 1, n2_split), (False, B, n2_whole)):
            key = (D, split, Bc)
            if key not in data:
                seed = 1000 * D + (7 if split else 11) + Bc
                data[key] = (_randn((Bc, N1, D), seed, dt), _randn((Bc, N2, D), seed + 1, dt))
            r, n = data[key]
            got_split, _ = knn_path(Bc, N1, N2, D, k, dt)
            assert got_split == split, (D, k, Bc, N2)
            for largest in (False, True):
                out = pp.knn(r, n, k=k, ord=ordv, largest=largest)
                for b in sorted({0, Bc - 1}):
                    check_knn(_np(out.values[b, rows]), out.indices[b, rows].cpu().numpy(), _np(r[b, rows]), _np(n[b]), k,
                              ordv, largest, dt, what=f"D={D} k={k} largest={largest} split={split} b={b}")
                reached.add(("3" if D == 3 else "general", K, largest, split))
    assert reached == {(c, K, l, s) for c in ("3", "general") for K in (1, 4, 8, 16, 32) for l in (False, True)
                       for s in (False, True)}
    print(f"\n{dt} ord={ordv}: reached {len(reached)} (D class, K, largest, split) combinations")


@pytest.mark.parametrize("dt", [F32, F64])
def test_knn_split_equals_unsplit_bit_for_bit(dt):
    """DESIGN §3.4: the merged per-split lists equal the unsplit search bit for bit.  The same queries and targets run
    once as B = 1 (split) and once as a batch of the queries replicated against the broadcast targets, large enough not
    to split."""
    N1, N2 = 300, 9000
    for D in (3, 7):
        r = _randn((1, N1, D), 50 + D, dt)
        n = _randn((1, N2, D), 60 + D, dt)
        for k in (1, 4, 8, 16, 32):
            nqb, _, _, _ = _knn_plan(1, N1, N2, D, k)
            B = -(-4 * _sms() // nqb)
            assert knn_path(1, N1, N2, D, k, dt)[0] and not knn_path(B, N1, N2, D, k, dt)[0]
            rb = r.expand(B, N1, D)
            for ordv in ORDS:
                for largest in (False, True):
                    a = pp.knn(r, n, k=k, ord=ordv, largest=largest)
                    b = pp.knn(rb, n, k=k, ord=ordv, largest=largest)
                    what = f"D={D} k={k} ord={ordv} largest={largest}"
                    assert torch.equal(b.values, a.values.expand_as(b.values)), what
                    assert torch.equal(b.indices, a.indices.expand_as(b.indices)), what


def _tie_scene(D, dt, chunk, N2=9000, seed=70):
    """Targets uniform in [0, 10)^D with bit-equal copies straddling split-chunk and 256-point tile edges, queries next
    to the copies (nearest ties) and copies far away at distinct distances (farthest ties)."""
    g = torch.Generator(device=DEV).manual_seed(seed + D)
    n = (torch.rand(N2, D, device=DEV, dtype=F64, generator=g) * 10).to(dt)
    near = [(chunk - 1, chunk), (255, 256), (511, 512), (chunk + 255, chunk + 256), (2 * chunk - 1, 2 * chunk),
            (5, chunk + 5, 2 * chunk + 5)]
    for grp in near:
        for j in grp[1:]:
            n[j] = n[grp[0]]
    far = [(chunk - 2, chunk + 1), (250, 3 * chunk + 1), (2 * chunk - 2, 2 * chunk + 1)]
    for m, (j1, j2) in enumerate(far):                 # farthest from everything, 100 > 90 > 80 along the diagonal
        n[j1] = n[j2] = 100.0 - 10.0 * m
    q = torch.stack([n[grp[0]] for grp in near])
    q[:, 0] += 2.0 ** -12
    return q[None], n[None], near, far


@pytest.mark.parametrize("dt", [F32, F64])
def test_knn_ties_across_split_and_tile_edges(dt):
    """Bit-equal targets on both sides of a split boundary and of 256-point tile edges: the lower index comes first in the
    split path and in the unsplit path, in both dtypes (the copies have bit-equal distances, so this is exact in fp32)."""
    for D in (3, 7):
        _, chunk = knn_path(1, 6, 9000, D, 4, dt)
        q, n, near, far = _tie_scene(D, dt, chunk)
        B = -(-4 * _sms() // _knn_plan(1, 6, 9000, D, 4)[0])
        for ordv in ORDS:
            for Bc in (1, B):
                split, _ = knn_path(Bc, q.shape[1], 9000, D, 4, dt)
                assert split == (Bc == 1)
                qq = q.expand(Bc, *q.shape[1:])
                out = pp.knn(qq, n, k=4, ord=ordv)
                idx = out.indices[-1].cpu().numpy()
                for r, grp in enumerate(near):
                    assert list(idx[r, :len(grp)]) == list(grp), (D, ordv, split, grp, idx[r])
                check_knn(_np(out.values[-1]), idx, _np(q[0]), _np(n[0]), 4, ordv, False, dt)
                assert knn_path(Bc, q.shape[1], 9000, D, 6, dt)[0] == (Bc == 1)
                far_out = pp.knn(qq, n, k=6, ord=ordv, largest=True).indices[-1].cpu().numpy()
                want = [j for pair in far for j in pair]
                assert (far_out == np.array(want)).all(), (D, ordv, split, far_out)


@pytest.mark.parametrize("dt", [F32, F64])
@pytest.mark.parametrize("ordv", ORDS)
def test_knn_non_finite_split_and_unsplit(dt, ordv):
    """A query with a NaN coordinate (one or all) gets index -1 and +inf (-inf with `largest`) in every slot; targets with
    a NaN coordinate never enter a list; with fewer finite targets than k the remaining slots are empty.  Split (B = 1)
    and unsplit (the queries replicated to a batch that does not split), D = 3 and general D."""
    N1, N2 = 300, 9000
    for D in (3, 7):
        _, chunk = knn_path(1, N1, N2, D, 5, dt)
        r = _randn((1, N1, D), 80 + D, dt)
        n = _randn((1, N2, D), 90 + D, dt)
        nan = float("nan")
        r[0, 0] = nan                                   # every coordinate
        r[0, 1, D - 1] = nan                            # one coordinate
        r[0, N1 - 1, 0] = nan
        for j in (0, 256, chunk - 1, chunk, N2 - 1):
            n[0, j] = nan
        for j in (1, 511, chunk + 1, 2 * chunk):
            n[0, j, (j % D)] = nan
        finite = np.flatnonzero(np.isfinite(_np(n[0])).all(1))
        sparse = torch.full_like(n, nan)                # 20 finite targets spread over the chunks
        keep = torch.arange(0, N2, N2 // 20, device=DEV)[:20]
        sparse[0, keep] = n[0, keep].nan_to_num(0.5)
        bad = [0, 1, N1 - 1]
        good = np.setdiff1d(_rows(N1), bad)
        for k in (5, 32):
            nqb = _knn_plan(1, N1, N2, D, k)[0]
            B = -(-4 * _sms() // nqb)
            for largest in (False, True):
                empty = -math.inf if largest else math.inf
                ref = None
                for Bc in (1, B):
                    assert knn_path(Bc, N1, N2, D, k, dt)[0] == (Bc == 1)
                    out = pp.knn(r.expand(Bc, N1, D), n, k=k, ord=ordv, largest=largest)
                    v, i = out.values[-1], out.indices[-1]
                    what = f"D={D} k={k} largest={largest} B={Bc}"
                    assert (i[bad] == -1).all() and (v[bad] == empty).all(), what
                    ig = i[good].cpu().numpy()
                    assert np.isin(ig, finite).all(), what
                    check_knn(_np(v[good]), np.searchsorted(finite, ig), _np(r[0, good]), _np(n[0, finite]), k, ordv,
                              largest, dt, what)
                    if ref is None:
                        ref = out
                    else:
                        assert torch.equal(out.values[-1], ref.values[0]) and torch.equal(out.indices[-1], ref.indices[0])
                    if k == 32:                         # fewer finite targets than k
                        out = pp.knn(r.expand(Bc, N1, D), sparse, k=32, ord=ordv, largest=largest)
                        v, i = out.values[-1], out.indices[-1]
                        assert (i[good][:, 20:] == -1).all() and (v[good][:, 20:] == empty).all(), what
                        assert np.isin(i[good][:, :20].cpu().numpy(), keep.cpu().numpy()).all(), what
                        assert (i[bad] == -1).all() and (v[bad] == empty).all(), what


def test_knn_largest_ord2_empty_slots_are_minus_inf():
    """Regression: an empty slot of a `largest` ord-2 list held sqrt(-inf) = NaN instead of -inf (the root of the
    squared distance was taken on the -inf sentinel)."""
    for dt in (F32, F64):
        r = torch.zeros(1, 2, 3, dtype=dt, device=DEV)
        r[0, 1, 0] = float("nan")
        n = torch.randn(1, 10, 3, dtype=dt, device=DEV)
        out = pp.knn(r, n, k=3, ord=2, largest=True)
        assert (out.indices[0, 1] == -1).all() and (out.values[0, 1] == -math.inf).all()
        assert (out.indices[0, 0] >= 0).all() and torch.isfinite(out.values[0, 0]).all()


def test_knn_ord_inf_nan_coordinate_gives_no_neighbour():
    """Regression: ord inf took max(|dx|, ...) with fmax, which drops NaN, so a point with one NaN coordinate got a finite
    distance from the others, and in general D a query or target NaN in every coordinate got distance 0 (the max
    started from 0)."""
    nan = float("nan")
    for dt in (F32, F64):
        for D in (3, 5):
            r = torch.zeros(1, 3, D, dtype=dt, device=DEV)
            r[0, 1, 0] = nan
            r[0, 2] = nan
            n = torch.ones(1, 4, D, dtype=dt, device=DEV) * torch.arange(1, 5, dtype=dt, device=DEV)[None, :, None]
            n[0, 0, D - 1] = nan
            n[0, 2] = nan
            out = pp.knn(r, n, k=3, ord=math.inf)
            assert out.indices[0, 0].tolist() == [1, 3, -1] and out.values[0, 0].tolist() == [2.0, 4.0, math.inf], (dt, D)
            assert (out.indices[0, 1:] == -1).all() and (out.values[0, 1:] == math.inf).all(), (dt, D)


@pytest.mark.parametrize("dt", [F32, F64])
def test_knn_filter_bucket16_vs_oracle(dt):
    """knn_filter with k = 8 and 15 (k + 1 in the 16 bucket): split (one cloud of 2300 points) and unsplit (a batch of 2
    clouds of 1200), against the fp64 oracle on every row whose k+1-th neighbour is unambiguous."""
    tol = 1e-6 if dt == F32 else 1e-12
    for shape, pdim, split in (((2300, 4), 3, True), ((2, 1200, 5), None, False)):
        x = _randn(shape, 31 + len(shape), dt)
        B = 1 if len(shape) == 2 else shape[0]
        p = _np(x).reshape(B, shape[-2], shape[-1])
        pd = pdim or shape[-1]
        for k in (8, 15):
            assert knn_path(B, shape[-2], shape[-2], pd, k + 1, dt)[0] == split
            for ordv in ORDS:
                got = pp.knn_filter(x, k, pdim=pdim, ord=ordv).reshape(B, shape[-2], shape[-1])
                for b in range(B):
                    d = np.sort(O.distances(p[b, :, :pd], p[b, :, :pd], ordv), -1)
                    clear = d[:, k + 1] - d[:, k] > 1e-5 * (1 + d[:, k])
                    assert clear.mean() > 0.99
                    want = PF.knn_filter(p[b], k, pdim, None, ordv)
                    np.testing.assert_allclose(_np(got[b])[clear], want[clear], rtol=0, atol=tol, err_msg=f"k={k} {ordv}")


# ---------------------------------------------------------------------------------------------------------------------
# radius mask, four queries per thread
# ---------------------------------------------------------------------------------------------------------------------
def _radius_q4(N):
    return -(-N // 1024) >= 2 * _sms()


def _mask_ok_tree(p, mask, nbr, radius, ordv, rel, sub):
    """mask on the rows `sub` equals the cKDTree count except at points within rel * radius of the radius."""
    from scipy.spatial import cKDTree
    tree = cKDTree(p)
    pn = {1: 1, 2: 2}.get(ordv, np.inf)
    lo = tree.query_ball_point(p[sub], radius * (1 - rel), p=pn, return_length=True) - 1 >= nbr
    hi = tree.query_ball_point(p[sub], radius * (1 + rel), p=pn, return_length=True) - 1 >= nbr
    m = mask.cpu().numpy()[sub]
    assert np.all(m[lo]) and not np.any(m[~hi]), (sub[lo & ~m][:5], sub[~hi & m][:5])
    return m


@pytest.mark.parametrize("dt", [F32, F64])
@pytest.mark.parametrize("ordv", ORDS)
def test_radius_mask_four_queries_per_thread(dt, ordv):
    """D = 3 at the smallest N that takes Q = 4 (ceil(N / 1024) = 2 SMs) and at 1e6 + 3 (a partly dead last CTA), with
    need 1, 16 and N + 5 (no query is ever satisfied, so every CTA scans every tile)."""
    rel = 1e-5 if dt == F32 else 1e-12
    for N in (1024 * (2 * _sms() - 1) + 7, 1000003):
        assert _radius_q4(N) and not _radius_q4(1024 * (2 * _sms() - 1))
        g = torch.Generator(device=DEV).manual_seed(N)
        pts = torch.rand(N, 3, device=DEV, dtype=F64, generator=g).to(dt)
        vol = {1: 4.0 / 3.0, 2: 4.0 * math.pi / 3.0}.get(ordv, 8.0)
        radius = (17.0 / (N * vol)) ** (1.0 / 3.0)   # about 16 neighbours inside the cube
        assert pp.nbr_filter(pts, 0, radius, ord=ordv, return_mask=True)[1].all()
        assert not pp.nbr_filter(pts, N + 4, radius, ord=ordv, return_mask=True)[1].any()
        mask = pp.nbr_filter(pts, 15, radius, ord=ordv, return_mask=True)[1]
        assert 0.1 < mask.float().mean().item() < 0.9
        rng = np.random.default_rng(N)
        sub = np.unique(np.r_[rng.integers(0, N, 20000), np.arange(N - 4096, N), np.arange(0, 1024)])
        _mask_ok_tree(_np(pts), mask, 15, radius, ordv, rel, sub)


@pytest.mark.parametrize("dt", [F32, F64])
def test_radius_mask_clusters_and_outliers_four_queries(dt):
    """Dense clusters (their CTAs stop after a few tiles) followed by 5 % uniform outliers (their CTAs scan every tile),
    on the four-query path."""
    rel = 1e-5 if dt == F32 else 1e-12
    N = 1024 * (2 * _sms() + 20) + 5
    g = torch.Generator(device=DEV).manual_seed(5)
    n_out = N // 20
    centres = torch.rand(300, 3, device=DEV, dtype=F64, generator=g) * 100
    dense = centres[torch.randint(0, 300, (N - n_out,), device=DEV, generator=g)]
    dense = dense + 0.3 * torch.randn(N - n_out, 3, device=DEV, dtype=F64, generator=g)
    dense = dense[torch.randperm(N - n_out, device=DEV, generator=g)]
    pts = torch.cat([dense, torch.rand(n_out, 3, device=DEV, dtype=F64, generator=g) * 100]).to(dt)
    assert _radius_q4(N)
    is_out = np.arange(N) >= N - n_out
    for ordv in ORDS:
        mask = pp.nbr_filter(pts, 15, 1.0, ord=ordv, return_mask=True)[1]
        m = mask.cpu().numpy()
        assert m[~is_out].mean() > 0.99 and m[is_out].mean() < 0.1
        sub = np.unique(np.r_[np.flatnonzero(is_out), np.random.default_rng(1).integers(0, N, 20000)])
        _mask_ok_tree(_np(pts), mask, 15, 1.0, ordv, rel, sub)


# ---------------------------------------------------------------------------------------------------------------------
# ICP: 256-thread CTAs of four queries, batches above 128
# ---------------------------------------------------------------------------------------------------------------------
class _Recording(pp.utils.ReduceToBason):
    """Not exactly ReduceToBason: ICP takes the host loop and calls step() every iteration."""

    def reset(self):
        super().reset()
        self.losses = []

    def step(self, loss):
        self.losses.append(loss.detach().double().cpu().numpy().reshape(-1).copy())
        super().step(loss)


class _Fixed(pp.utils.ReduceToBason):
    """A fixed number of host-loop iterations."""

    def __init__(self, steps):
        super().__init__(steps, patience=10 ** 9, tol=-1.0)


def _mats(se3):
    return O.se3_to_mat(_np(se3.tensor() if hasattr(se3, "tensor") else se3)).reshape(-1, 3, 4)


def _rigid(rng, B, angle, shift):
    ax = rng.standard_normal((B, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    th = angle * rng.uniform(0.5, 1.0, (B, 1))
    q = np.c_[ax * np.sin(th / 2), np.cos(th / 2)]
    R = np.stack([O.quat2mat(x) for x in q])
    return R, shift * rng.uniform(-1, 1, (B, 3))


def _jittered_grid(rng, side, spacing, jitter=0.2):
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    g = (g - (side - 1) / 2) * spacing
    return g + rng.uniform(-jitter, jitter, g.shape)


def _batch_scene(B, seed, slow=True):
    """B jittered 9^3 grids (spacing 1.5: points at least 1.1 apart), each moved by a small rigid motion plus 0.01 noise:
    every nearest neighbour is unambiguous.  Element 0 gets a larger motion and converges over many more steps, so the
    batch-wide stop rule follows it."""
    rng = np.random.default_rng(seed)
    src = np.stack([_jittered_grid(rng, 9, 1.5) for _ in range(B)])
    R, t = _rigid(rng, B, 0.02, 0.05)
    if slow:
        R[0], t[0] = _rigid(rng, 1, 0.2, 0.0)[0][0], np.array([0.4, -0.3, 0.2])
    tgt = np.einsum("bij,bnj->bni", R, src) + t[:, None] + 0.01 * rng.standard_normal(src.shape)
    return src, tgt


def _run(src, tgt, dt, ordv, init=None, stepper=None):
    st = stepper if stepper is not None else pp.utils.ReduceToBason(60)
    it = None if init is None else pp.SE3(torch.from_numpy(init).to(DEV, dt))
    out = pp.module.ICP(stepper=st)(torch.from_numpy(src).to(DEV, dt), torch.from_numpy(tgt).to(DEV, dt), ord=ordv, init=it)
    return out, st


def check_icp(src, tgt, dt, ordv, init=None, what=""):
    """Host loop against the fp64 oracle (transform, per-step losses, fp64 step count) and the device-decided loop
    against the host loop (same steps, bit-identical transform)."""
    f32 = dt == F32
    s = src.astype(np.float32).astype(np.float64) if f32 else src
    t = tgt.astype(np.float32).astype(np.float64) if f32 else tgt
    i0 = None if init is None else (init.astype(np.float32).astype(np.float64) if f32 else init)
    out, st = _run(s, t, dt, ordv, i0, _Recording(60))
    A, L, _ = O.icp(s, t, None if i0 is None else O.se3_to_mat(i0), ordv, 60, eps=O.KABSCH_EPS[np.float32 if f32 else np.float64],
                    matcher="kdtree")
    got = _mats(out)
    np.testing.assert_allclose(got, A, atol=2e-5 if f32 else 1e-9, err_msg=what)
    n = min(len(st.losses), len(L))
    tol = 2e-5 if f32 else 1e-9
    np.testing.assert_allclose(np.array(st.losses[:n]), L[:n].reshape(n, -1), rtol=tol, atol=tol, err_msg=what)
    if f32:
        print(f"\n{what}: fp32 steps {st.steps}, fp64 oracle {len(L)}")
    else:
        assert st.steps == len(L), what
    out2, st2 = _run(s, t, dt, ordv, i0)
    assert st2.steps == st.steps and torch.equal(out2.tensor(), out.tensor()), what
    return st.steps


@pytest.mark.parametrize("dt", [F32, F64])
@pytest.mark.parametrize("ordv", ORDS)
def test_icp_big_ctas_batch_vs_oracle(dt, ordv):
    """B = 2 SMs + 16 clouds of 729 points: the 256-thread CTAs of four queries (nx = 1) and an update launch of more
    than 128 CTAs, whose last CTA loops over the batch for the stop rule."""
    B = 2 * _sms() + 16
    src, tgt = _batch_scene(B, 7 + ORDS.index(ordv))
    assert icp_nx(B, 729) == 1 and icp_nx(1, 729) == 6 and B > 128
    steps = check_icp(src, tgt, dt, ordv, what=f"{dt} ord={ordv}")
    assert steps >= 10                                   # decided by the slow element


@pytest.mark.parametrize("dt", [F32, F64])
def test_icp_big_ctas_broadcast_and_init(dt):
    """Stride 0 on either side (one source against per-element targets and the reverse) and a per-element init (stride
    7), on the four-query path."""
    B = 2 * _sms() + 16
    rng = np.random.default_rng(3)
    one = _jittered_grid(rng, 9, 1.5)[None]
    R, t = _rigid(rng, B, 0.02, 0.05)
    many = np.einsum("bij,nj->bni", R, one[0]) + t[:, None] + 0.01 * rng.standard_normal((B, 729, 3))
    assert icp_nx(B, 729) == 1
    check_icp(one, many, dt, 2, what="broadcast source")
    check_icp(many, one, dt, 2, what="broadcast target")
    src, tgt = _batch_scene(B, 4, slow=False)
    Ri, ti = _rigid(rng, B, 0.01, 0.02)
    init = np.concatenate([ti, np.stack([_mat2quat(r) for r in Ri])], 1)
    check_icp(src, tgt, dt, 1, init=init, what="per-element init")


def _mat2quat(R):
    w = math.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])


@pytest.mark.parametrize("dt", [F32, F64])
def test_icp_big_ctas_large_source(dt):
    """B = 4 sources of 70 000 points (nx = 69 CTAs of 1024 each, the last one partly dead) against 17^3 = 4913-point
    targets; the fp64 oracle matches with a k-d tree.  Each source point lies within 0.2 of its target point, which are
    at least 1.6 apart."""
    rng = np.random.default_rng(11)
    tgt = np.stack([_jittered_grid(rng, 17, 2.0) for _ in range(4)])
    Ns = 70000
    src0 = tgt[:, np.arange(Ns) % tgt.shape[1]] + 0.05 * np.clip(rng.standard_normal((4, Ns, 3)), -3, 3)
    R, t = _rigid(rng, 4, 0.01, 0.05)
    src = np.einsum("bji,bnj->bni", R, src0 - t[:, None])          # tgt ~ R src + t
    assert icp_nx(4, Ns) == 69
    for ordv in (2, math.inf):
        check_icp(src, tgt, dt, ordv, what=f"large source ord={ordv}")


def test_icp_big_batch_equals_elements_alone():
    """fp64: each element run alone (B = 1, 128-thread CTAs) and inside the big batch (256 x 4) agree to 1e-12 after a
    fixed 8 host-loop iterations: same matches, partial sums reduced in another order."""
    B = 2 * _sms() + 16
    src, tgt = _batch_scene(B, 21)
    assert icp_nx(B, 729) == 1 and icp_nx(1, 729) == 6
    for ordv in ORDS:
        big, _ = _run(src, tgt, F64, ordv, stepper=_Fixed(8))
        Ab = _mats(big)
        for b in (0, 1, B // 2, B - 1):
            one, st = _run(src[b:b + 1], tgt[b:b + 1], F64, ordv, stepper=_Fixed(8))
            assert st.steps == 8
            np.testing.assert_allclose(_mats(one)[0], Ab[b], rtol=0, atol=1e-12, err_msg=f"ord={ordv} b={b}")
