"""pp.svdstf and the point-cloud filters (csrc/knn.cu radius mask, csrc/voxel.cu) against the reference goldens
(tests/golden/pcfilter.npz, oracle/make_golden_pcfilter.py) and the numpy oracle (oracle/pcfilter_oracle.py)."""
import math
import os

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from pypose_b200.function import geometry as G
from oracle import pcfilter_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "pcfilter.npz"))


def _names(prefix):
    return sorted({k.split("/")[1] for k in GOLD.files if k.startswith(prefix + "/")})


def _ord(v):
    return math.inf if int(v) == -1 else int(v)


def _nbr_case(name):
    p = f"nbr/{name}/"
    nbr, radius, pdim, o = GOLD[p + "args"]
    return GOLD[p + "points"], int(nbr), float(radius), int(pdim) or None, _ord(o), GOLD[p + "mask"]


def _knnf_case(name):
    p = f"knnf/{name}/"
    k, pdim, radius, o = GOLD[p + "args"]
    return GOLD[p + "points"], int(k), int(pdim) or None, None if radius < 0 else float(radius), _ord(o), GOLD[p + "out"]


def _voxel_case(name):
    p = f"voxel/{name}/"
    return GOLD[p + "points"], [float(v) for v in GOLD[p + "voxel"]], GOLD[p + "out"]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: oracle vs goldens, svdstf / random_filter, the ord-2 threshold, the key planner, argument checks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", _names("voxel"))
def test_oracle_voxel_is_bit_identical_to_reference(name):
    pts, vox, out = _voxel_case(name)
    got = O.voxel_centroids(pts, vox)
    assert got.dtype == out.dtype and np.array_equal(got, out)


@pytest.mark.parametrize("name", _names("nbr"))
def test_oracle_nbr_mask_matches_reference(name):
    pts, nbr, radius, pdim, o, mask = _nbr_case(name)
    np.testing.assert_array_equal(O.nbr_mask(pts, nbr, radius, pdim, o), mask)


@pytest.mark.parametrize("name", _names("knnf"))
def test_oracle_knn_filter_matches_reference(name):
    pts, k, pdim, radius, o, out = _knnf_case(name)
    np.testing.assert_allclose(O.knn_filter(pts, k, pdim, radius, o), out, rtol=0, atol=1e-12 if out.dtype == np.float64 else 1e-6)


@pytest.mark.parametrize("name", _names("svdstf"))
def test_svdstf_matches_reference_on_cpu(name):
    p = f"svdstf/{name}/"
    src, tgt, ws = GOLD[p + "source"], GOLD[p + "target"], bool(GOLD[p + "with_scale"])
    tol = 1e-6 if src.dtype == np.float32 else 1e-12
    np.testing.assert_allclose(O.svdstf(src, tgt, ws), GOLD[p + "matrix"], atol=tol)
    out = pp.svdstf(torch.from_numpy(src), torch.from_numpy(tgt), with_scale=ws)
    assert out.ltype == pp.Sim3_type
    np.testing.assert_allclose(out.tensor().numpy(), GOLD[p + "out"], atol=tol)


def test_random_filter_shapes_and_rows_on_cpu():
    for B, N, num, D in GOLD["random/shapes"]:
        pts = torch.randn(int(B), int(N), int(D))
        out = pp.random_filter(pts, int(num))
        assert out.shape == (B, num, D)
        # the same rows for every batch element, without repetition
        rows = [int((pts[0] == r).all(-1).nonzero()) for r in out[0]]
        assert len(set(rows)) == num and torch.equal(out, pts[:, rows])
    torch.manual_seed(5)
    a = pp.random_filter(torch.arange(20.).view(10, 2), 4)
    torch.manual_seed(5)
    assert torch.equal(a, pp.random_filter(torch.arange(20.).view(10, 2), 4))
    with pytest.raises(ValueError):
        pp.random_filter(torch.randn(10, 3), 11)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_sq_threshold_is_the_largest_with_root_below_radius(dtype):
    ft = np.float32 if dtype == torch.float32 else np.float64
    rng = np.random.default_rng(1)
    radii = np.concatenate([10.0 ** rng.uniform(-6, 6, 3000), [0.0, 1.0, 2.0, 1.5, 3.0, 1e-30]])
    for r in radii:
        t = ft(G._sq_threshold(float(r), dtype))
        rr = ft(r)
        assert np.sqrt(t) <= rr < np.sqrt(np.nextafter(t, ft(np.inf))), (r, t)
    assert G._sq_threshold(-1.0, dtype) < 0 and G._sq_threshold(math.inf, dtype) == math.inf


def test_voxel_plan_preserves_lexicographic_order_and_splits_groups():
    rng = np.random.default_rng(2)
    for lo, hi in (([0, -5, 0], [9, 0, 1000]), ([0] * 3, [2 ** 30] * 3), ([0, 0], [0, 7]), ([-(2 ** 61), 0], [0, 2 ** 61])):
        layout, bits = G._voxel_plan(lo, hi)
        widths = [int(h - l).bit_length() for l, h in zip(lo, hi)]
        assert sum(bits) == sum(widths) and all(0 <= b <= 64 for b in bits)
        assert len(bits) == (1 if sum(widths) <= 64 else 2)
        assert [g for g, _ in layout] == sorted(g for g, _ in layout)          # dimensions stay in order
        c = np.stack([rng.integers(l, h + 1, 400) for l, h in zip(lo, hi)], 1)
        c[200:] = c[:200]                                                      # equal rows too
        keys = [tuple(sum((int(row[d]) - lo[d]) << layout[d][1] for d in range(len(lo)) if layout[d][0] == g)
                      for g in range(len(bits))) for row in c]
        assert all(k < 2 ** 64 for ks in keys for k in ks)
        by_key = sorted(range(len(c)), key=lambda i: (keys[i], i))
        by_coord = sorted(range(len(c)), key=lambda i: (tuple(c[i]), i))
        assert by_key == by_coord


def test_voxel_ranges_replicate_float_ops_and_refuse_huge_extents():
    lo, hi = G._voxel_ranges(np.array([0.0, -1.0], np.float32), np.array([1.0, 1.0], np.float32),
                             np.array([0.1, -0.3], np.float32), torch.float32)
    assert lo == [0, -6] and hi == [int(np.float32(1.0) / np.float32(0.1)), 0]
    with pytest.raises(ValueError):
        G._voxel_ranges(np.array([0.0]), np.array([1.0]), np.array([1e-19]), torch.float64)
    with pytest.raises(ValueError):
        G._voxel_ranges(np.array([0.0]), np.array([np.inf]), np.array([1.0]), torch.float64)


def test_argument_validation():
    p = torch.randn(10, 3)
    with pytest.raises(ValueError):
        pp.nbr_filter(p, 2, 1.0, ord=3)
    with pytest.raises(ValueError):
        pp.nbr_filter(p, 2, 1.0, pdim=4)
    with pytest.raises(ValueError):
        pp.nbr_filter(p[None], 2, 1.0)
    with pytest.raises(ValueError):
        pp.knn_filter(p, 31)                          # k + 1 > 32
    with pytest.raises(ValueError):
        pp.knn_filter(p, 10)                          # k + 1 > N
    with pytest.raises(ValueError):
        pp.knn_filter(p, 2, ord=0)
    with pytest.raises(ValueError):
        pp.knn_filter(p[None], 2, radius=1.0)
    with pytest.raises(ValueError):
        pp.voxel_filter(p, [0.1, 0.0])
    with pytest.raises(ValueError):
        pp.voxel_filter(p, [0.1] * 4)
    with pytest.raises(ValueError):
        pp.voxel_filter(p[None], [0.1])


def test_cpu_tensors_raise_on_the_gpu_paths():
    p = torch.randn(10, 3)
    for f in (lambda: pp.nbr_filter(p, 2, 1.0), lambda: pp.knn_filter(p, 2), lambda: pp.knn_filter(p, 2, radius=1.0),
              lambda: pp.voxel_filter(p, [0.5, 0.5, 0.5]), lambda: pp.voxel_filter(p, [0.5], random=True)):
        with pytest.raises(NotImplementedError, match="CPU"):
            f()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
DEV = "cuda"


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _names("voxel"))
def test_voxel_filter_is_bit_identical_to_reference(name):
    pts, vox, out = _voxel_case(name)
    got = pp.voxel_filter(_cuda(pts), vox)
    assert got.dtype == _cuda(out).dtype and torch.equal(got, _cuda(out))


def _cloud(n, dtype, seed, scale=10.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.rand(n, 3, device=DEV, dtype=torch.float64, generator=g) * scale).to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,voxel", [(1000, [0.7, 0.9, 0.8]), (200003, [0.2, 0.25, 0.3]), (2000000, [0.09, 0.1, 0.11]),
                                     (50000, [-0.5, 2.0, 0.3])])
def test_voxel_filter_matches_oracle(dtype, n, voxel):
    pts = _cloud(n, dtype, n)
    got = pp.voxel_filter(pts, voxel)
    ref = O.voxel_centroids(pts.cpu().numpy(), voxel)
    assert torch.equal(got, _cuda(ref))
    assert torch.equal(pp.voxel_filter(pts, voxel), got)                     # bit-reproducible


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_voxel_filter_special_clouds(dtype):
    # more than 64 key bits (two groups): ~2^30 voxels per dimension
    pts = _cloud(30000, dtype, 3, scale=1.0)
    pts[:15000] = pts[15000:]                                                 # every voxel twice
    vox = [1e-9, 2e-9, 1.5e-9]
    layout, bits = G._voxel_plan(*G._voxel_ranges(pts.min(0).values.cpu().numpy(), pts.max(0).values.cpu().numpy(),
                                                  np.array(vox, np.float32).astype(pts.cpu().numpy().dtype), dtype))
    assert len(bits) == 2
    assert torch.equal(pp.voxel_filter(pts, vox), _cuda(O.voxel_centroids(pts.cpu().numpy(), vox)))
    # the whole cloud in one voxel
    one = _cloud(300000, dtype, 4, scale=1.0)
    got = pp.voxel_filter(one, [2.0, 2.0])
    assert got.shape == (1, 3) and torch.equal(got, _cuda(O.voxel_centroids(one.cpu().numpy(), [2.0, 2.0])))
    # non-contiguous input, vdim < D
    wide = _cloud(20000, dtype, 5).repeat(1, 2)[:, 1:]                        # (N, 5) with a row stride of 6
    assert not wide.is_contiguous()
    assert torch.equal(pp.voxel_filter(wide, [0.5, 0.6]), _cuda(O.voxel_centroids(wide.cpu().numpy(), [0.5, 0.6])))
    assert pp.voxel_filter(one[:0], [1.0]).shape == (0, 3)


@pytest.mark.gpu
def test_voxel_filter_random_members_and_seed():
    pts = _cloud(50000, torch.float32, 6)
    vox = [0.8, 0.8, 0.8]
    order, start, vid = O.voxel_segments(pts.cpu().numpy(), vox)
    torch.manual_seed(3)
    a = pp.voxel_filter(pts, vox, random=True)
    torch.manual_seed(3)
    b = pp.voxel_filter(pts, vox, random=True)
    assert torch.equal(a, b) and a.shape == (len(start) - 1, 3)
    # every output row is a member of the voxel at its position
    cen = O.voxel_centroids(pts.cpu().numpy(), vox)
    rows = a.cpu().numpy()
    member_vox = O.voxel_coords(np.concatenate([pts.cpu().numpy(), rows]), vox)[len(order):]
    all_vox = O.voxel_coords(pts.cpu().numpy(), vox)[order[start[:-1]]]
    assert np.array_equal(member_vox, all_vox)
    assert cen.shape == rows.shape
    # one point per voxel: the random mode returns (M, D), also for a single voxel
    assert pp.voxel_filter(pts[:5], [100.0], random=True).shape == (1, 3)


@pytest.mark.gpu
def test_voxel_filter_random_is_uniform():
    counts = np.array([1, 2, 3, 5, 8])
    x = np.concatenate([np.full(c, i, np.float64) for i, c in enumerate(counts)]) * 10
    pts = torch.from_numpy(np.stack([x, np.arange(len(x)) * 0.01, np.zeros(len(x))], 1)).to(DEV)
    R = 4000
    seen = np.zeros(len(x), np.int64)
    torch.manual_seed(0)
    for _ in range(R):
        out = pp.voxel_filter(pts, [5.0], random=True)
        idx = torch.round(out[:, 1] / 0.01).long().cpu().numpy()
        seen[idx] += 1
    p = np.concatenate([np.full(c, 1.0 / c) for c in counts])
    sigma = np.sqrt(R * p * (1 - p))
    assert np.all(np.abs(seen - R * p) <= 5 * sigma + 1e-9), (seen, R * p)


@pytest.mark.gpu
def test_voxel_filter_gradcheck():
    g = torch.Generator().manual_seed(8)
    cells = torch.randint(0, 4, (40, 3), generator=g).double()
    pts = torch.cat([torch.zeros(1, 4, dtype=torch.float64),
                     torch.cat([(cells + 0.5 + 0.3 * (torch.rand(40, 3, generator=g, dtype=torch.float64) - 0.5)) * 0.5,
                                torch.randn(40, 1, generator=g, dtype=torch.float64)], 1)]).to(DEV).requires_grad_()
    assert torch.autograd.gradcheck(lambda p: pp.voxel_filter(p, [0.5, 0.5, 0.5]), (pts,))


def _mask_ok(pts, nbr, radius, pdim, ordv, mask, rel):
    """Equal to the brute-force oracle except at points with a distance within rel * radius of the radius."""
    lo = O.radius_counts(pts, radius * (1 - rel), pdim, ordv) - 1 >= nbr
    hi = O.radius_counts(pts, radius * (1 + rel), pdim, ordv) - 1 >= nbr
    m = mask.cpu().numpy()
    assert np.all(m[lo]) and not np.any(m[~hi]), (np.flatnonzero(lo & ~m), np.flatnonzero(~hi & m))


@pytest.mark.gpu
@pytest.mark.parametrize("name", _names("nbr"))
def test_nbr_filter_matches_reference(name):
    pts, nbr, radius, pdim, o, mask = _nbr_case(name)
    out, got = pp.nbr_filter(_cuda(pts), nbr, radius, pdim=pdim, ord=o, return_mask=True)
    assert torch.equal(got.cpu(), torch.from_numpy(mask)) and torch.equal(out, _cuda(pts)[got])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D,pdim,ordv", [(3, None, 2), (3, None, 1), (3, None, math.inf), (5, 4, 2), (4, 2, 1)])
def test_nbr_filter_random_clouds(dtype, D, pdim, ordv):
    g = torch.Generator(device=DEV).manual_seed(D * 10 + (pdim or 0))
    pts = (torch.rand(3000, D, device=DEV, dtype=torch.float64, generator=g) * 4).to(dtype)
    rel = 1e-5 if dtype == torch.float32 else 1e-12
    for nbr, radius in ((0, 0.1), (3, 0.35), (10, 0.5), (-1, 0.2)):
        mask = pp.nbr_filter(pts, nbr, radius, pdim=pdim, ord=ordv, return_mask=True)[1]
        _mask_ok(pts.cpu().numpy(), nbr, radius, pdim, ordv, mask, rel)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_nbr_filter_early_exit_and_full_scan(dtype):
    """Dense clusters (their CTAs stop after a few tiles) and sparse outliers at the end (their CTAs scan every tile)."""
    g = torch.Generator(device=DEV).manual_seed(9)
    centres = torch.rand(20, 3, device=DEV, dtype=torch.float64, generator=g) * 100
    dense = centres.repeat_interleave(2400, 0) + 0.3 * torch.randn(48000, 3, device=DEV, dtype=torch.float64, generator=g)
    dense = dense[torch.randperm(48000, device=DEV, generator=g)]
    sparse = torch.rand(2000, 3, device=DEV, dtype=torch.float64, generator=g) * 100
    pts = torch.cat([dense, sparse]).to(dtype)
    mask = pp.nbr_filter(pts, 20, 1.0, return_mask=True)[1]
    assert mask[:48000].float().mean() > 0.99 and mask[48000:].float().mean() < 0.1
    from scipy.spatial import cKDTree
    p = pts.cpu().numpy().astype(np.float64)
    tree = cKDTree(p)
    rel = 1e-5 if dtype == torch.float32 else 1e-12
    lo = tree.query_ball_point(p, 1.0 * (1 - rel), return_length=True) - 1 >= 20
    hi = tree.query_ball_point(p, 1.0 * (1 + rel), return_length=True) - 1 >= 20
    m = mask.cpu().numpy()
    assert np.all(m[lo]) and not np.any(m[~hi])


@pytest.mark.gpu
@pytest.mark.parametrize("name", _names("knnf"))
def test_knn_filter_matches_reference(name):
    pts, k, pdim, radius, o, out = _knnf_case(name)
    got = pp.knn_filter(_cuda(pts), k, pdim=pdim, radius=radius, ord=o)
    tol = 1e-6 if out.dtype == np.float32 else 1e-12
    np.testing.assert_allclose(got.cpu().numpy(), out, rtol=0, atol=tol)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_knn_filter_batched_and_radius_vs_oracle(dtype):
    g = torch.Generator(device=DEV).manual_seed(10)
    x = torch.randn(3, 2, 500, 4, device=DEV, dtype=torch.float64, generator=g).to(dtype)
    tol = 1e-6 if dtype == torch.float32 else 1e-12
    for k, pdim, o in ((5, 3, 2), (31, None, 1), (7, 2, math.inf)):
        got = pp.knn_filter(x, k, pdim=pdim, ord=o)
        assert got.shape == x.shape
        for i in range(3):
            for j in range(2):
                assert torch.equal(got[i, j], pp.knn_filter(x[i, j], k, pdim=pdim, ord=o))
        np.testing.assert_allclose(got.cpu().numpy(), O.knn_filter(x.cpu().numpy(), k, pdim, None, o), rtol=0, atol=tol)
    # with a radius: outliers anywhere in the cloud; neighbours from the full cloud
    y = torch.cat([torch.randn(900, 3, device=DEV, dtype=torch.float64, generator=g) * 0.5,
                   torch.rand(100, 3, device=DEV, dtype=torch.float64, generator=g) * 40 - 20])
    y = y[torch.randperm(1000, device=DEV, generator=g)].to(dtype)
    got = pp.knn_filter(y, 4, radius=0.4)
    ref = O.knn_filter(y.cpu().numpy(), 4, None, 0.4, 2)
    assert got.shape == ref.shape and 0 < got.shape[0] < 1000
    np.testing.assert_allclose(got.cpu().numpy(), ref, rtol=0, atol=tol)
