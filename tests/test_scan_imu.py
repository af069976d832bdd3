"""Scans and IMU preintegration: oracle pinned to the reference goldens; host logic on CPU; kernels on GPU."""
import os

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import scan_oracle as S
from oracle import lie_oracle as O

GROUPS = ["SO3", "SE3", "RxSO3", "Sim3"]
CTOR = {"SO3": pp.SO3, "SE3": pp.SE3, "RxSO3": pp.RxSO3, "Sim3": pp.Sim3}
U32 = 2.0 ** -24                       # fp32 unit roundoff


def _within(what, err, scale, tol):
    """err <= tol * scale, with both numbers in the message."""
    assert err <= tol * scale, f"{what}: max error {err:.3e} > {tol:.3e} x scale {scale:.3e}"


def _scan_logstep(grp, x, left):
    """Inclusive group-product scan of x (B, L, D) in fp64 by log-step doubling (Hillis-Steele): after the round with
    offset s, y_i holds the product of rows max(0, i - 2s + 1) .. i.  ceil(log2 L) vectorised O.mul passes, so it serves
    as the fp64 truth at lengths where the sequential S.cumprod is too slow."""
    y = np.array(x, dtype=np.float64)
    B, L, D = y.shape
    s = 1
    while s < L:
        early, late = y[:, :-s].reshape(-1, D), y[:, s:].reshape(-1, D)
        y[:, s:] = (O.mul(grp, late, early) if left else O.mul(grp, early, late)).reshape(B, L - s, D)
        s *= 2
    return y


def _scan_f32_tol(B, L):
    """fp32 bound of the scans relative to 1 + max|truth|: unit roundoff u times
      4 x the sequential combines an output passes through on the route _cumprod_cuda takes for (B, L) (csrc/scan.cu;
        kScanThreads = 128, CH = 8 rows per thread, 1024-row tiles; 4u covers one quaternion product / rotated
        translation):
          in the tile    CH thread rows + 5 warp-shuffle levels + 3 warp totals of the 4-warp prefix + 2 (exclusive
                         prefix, prefix x row);
          single pass    + one carry per preceding tile (cumprod_kernel walks the tiles in order);
          time split     + the tile-prefix kernel: 5 + 5 shuffle levels (tile aggregates, warp totals) + 2 + one carry
                         per 1024-tile round;
      + L / 4: an output is the product of up to L rounded factors and their errors need not cancel.  A product of
        scales within 1e-5 of 1 (RxSO3 / Sim3) drifts by ~0.06 u per factor in fp32, whatever the order (a sequential
        numpy fp32 cumprod drifts the same way), so the depth term alone does not bound it.
    Measured on an H100 (DESIGN.md §4): <= 256 u at L = 4097, <= 7.4e4 u at L = 1.2e6 (RxSO3)."""
    tile = 1024
    nt = -(-L // tile)
    depth = 8 + 5 + 3 + 2
    if B < 2 * torch.cuda.get_device_properties(0).multi_processor_count and L >= 4 * tile:
        depth += 5 + 5 + 2 + -(-nt // 1024)
    else:
        depth += nt
    return U32 * (4 * depth + L / 4)


@pytest.mark.parametrize("grp", GROUPS)
def test_oracle_cumprod_matches_reference(golden_scan, grp):
    x = golden_scan[f"cumprod/{grp}/in"]
    np.testing.assert_allclose(S.cumprod(grp, x, True), golden_scan[f"cumprod/{grp}/left"], atol=1e-12)
    np.testing.assert_allclose(S.cumprod(grp, x, False), golden_scan[f"cumprod/{grp}/right"], atol=1e-12)


@pytest.mark.parametrize("tag", ["free", "rot"])
def test_oracle_imu_matches_reference(golden_scan, tag):
    g = golden_scan
    rot = g["imu/rot"] if tag == "rot" else None
    outs = S.imu_integrate(g["imu/dt"], g["imu/gyro"], g["imu/acc"], rot, g["imu/init_rot"])
    for name, o in zip(("a", "Dp", "Dv", "Dr", "Dt", "w"), outs):
        np.testing.assert_allclose(o, g[f"imu/{tag}/inte/{name}"], atol=1e-12, err_msg=name)


def _dev(request):
    return "cuda" if request.node.get_closest_marker("gpu") else "cpu"


def _check_cumprod_api(golden_scan, grp, dev, tol):
    x = CTOR[grp](torch.from_numpy(golden_scan[f"cumprod/{grp}/in"]).to(dev))
    for left, key in ((True, "left"), (False, "right")):
        y = x.cumprod(dim=1, left=left)
        assert isinstance(y, pp.LieTensor) and y.ltype is x.ltype
        np.testing.assert_allclose(y.tensor().cpu().numpy(), golden_scan[f"cumprod/{grp}/{key}"], atol=tol)
        np.testing.assert_allclose(pp.cummul(x, 1, left).tensor().cpu().numpy(), golden_scan[f"cumprod/{grp}/{key}"], atol=tol)
    # scan along dim 0 of a (L, B, D) view, in place variant, and the explicit 4-factor product
    # (reference tests/basics/test_ops.py:15-57)
    xt = CTOR[grp](x.tensor().transpose(0, 1).contiguous())
    y0 = xt.cumprod(dim=0, left=True)
    np.testing.assert_allclose(y0.tensor().transpose(0, 1).cpu().numpy(), golden_scan[f"cumprod/{grp}/left"], atol=tol)
    four = x[:, :4]
    last = four.cumprod(dim=1, left=True)[:, -1]
    ref = four[:, 3] @ four[:, 2] @ four[:, 1] @ four[:, 0]
    np.testing.assert_allclose(last.tensor().cpu().numpy(), ref.tensor().cpu().numpy(), atol=tol)
    z = x.clone()
    z.cumprod_(dim=1, left=False)
    np.testing.assert_allclose(z.tensor().cpu().numpy(), golden_scan[f"cumprod/{grp}/right"], atol=tol)


@pytest.mark.parametrize("grp", GROUPS)
def test_cumprod_api_cpu(golden_scan, grp):
    _check_cumprod_api(golden_scan, grp, "cpu", 1e-12)


def test_cumops_generic_equals_cumsum():
    # reference tests/lietensor/test_lietensor.py:214-221
    for n in (1, 2, 3, 17, 100, 257):
        x = torch.randn(n, 3, dtype=torch.float64)
        torch.testing.assert_close(pp.cumops(x, 0, lambda a, b: a + b), torch.cumsum(x, 0))


def _check_imu_module(golden_scan, dev, tol):
    g = golden_scan
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    init = {"pos": t("imu/init_pos"), "rot": pp.SO3(t("imu/init_rot")), "vel": t("imu/init_vel")}
    for tag in ("free", "rot"):
        m = pp.module.IMUPreintegrator(prop_cov=True, reset=True).double().to(dev)
        kw = {"rot": pp.SO3(t("imu/rot"))} if tag == "rot" else {}
        out = m(t("imu/dt"), t("imu/gyro"), t("imu/acc"), init_state=init, **kw)
        for k in ("rot", "vel", "pos", "cov"):
            v = out[k].tensor() if isinstance(out[k], pp.LieTensor) else out[k]
            np.testing.assert_allclose(v.cpu().numpy(), g[f"imu/{tag}/out/{k}"], atol=tol, rtol=tol, err_msg=f"{tag}/{k}")
        # fused integrate+predict path (prop_cov=False)
        m2 = pp.module.IMUPreintegrator(prop_cov=False, reset=True).double().to(dev)
        out2 = m2(t("imu/dt"), t("imu/gyro"), t("imu/acc"), init_state=init, **kw)
        for k in ("rot", "vel", "pos"):
            v = out2[k].tensor() if isinstance(out2[k], pp.LieTensor) else out2[k]
            np.testing.assert_allclose(v.cpu().numpy(), g[f"imu/{tag}/out/{k}"], atol=tol, rtol=tol, err_msg=f"fused {tag}/{k}")
        assert out2["cov"] is None


def test_imu_module_cpu(golden_scan):
    _check_imu_module(golden_scan, "cpu", 1e-10)


def test_imu_docstring_known_answer():
    """imu_preintegrator.py:28-53: one sample, dt = 0.002, known identity rotation (rot/vel/pos; the
    docstring's printed cov is stale, SURVEY.md §4)."""
    p = pp.module.IMUPreintegrator(torch.zeros(3), pp.identity_SO3(), torch.zeros(3), prop_cov=False, reset=True)
    out = p(torch.tensor([0.002]), torch.tensor([0.1, 0.1, 0.1]), torch.tensor([0.1, 0.1, 0.1]), pp.identity_SO3())
    torch.testing.assert_close(out["rot"].tensor().flatten(), torch.tensor([1e-4, 1e-4, 1e-4, 1.0]), atol=1e-7, rtol=0)
    torch.testing.assert_close(out["vel"].flatten(), torch.tensor([0.0002, 0.0002, -0.0194]), atol=5e-5, rtol=0)
    torch.testing.assert_close(out["pos"].flatten(), torch.tensor([2.0e-07, 2.0e-07, -1.9420e-05]), atol=5e-9, rtol=0)


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("grp", GROUPS)
def test_cumprod_api_gpu(golden_scan, grp):
    _check_cumprod_api(golden_scan, grp, "cuda", 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("grp", GROUPS)
@pytest.mark.parametrize("L", [1, 2, 31, 32, 33, 127, 128, 129, 1000, 4097])
@pytest.mark.parametrize("dt", [torch.float64, torch.float32], ids=["f64", "f32"])
def test_cumprod_kernel_vs_oracle_lengths(grp, L, dt):
    """cumprod_kernel (and, at L = 4097, the time-split route) against the sequential oracle; fp64 at 1e-11, fp32 at the
    bound derived from the combine depth (_scan_f32_tol)."""
    from tests.util import rand_group
    rng = np.random.default_rng(L)
    x = rand_group(rng, grp, 3 * L, tmax=0.3, t_sigma=0.1, s_sigma=0.02).reshape(3, L, -1)
    xd = torch.from_numpy(x).to(dt).cuda()
    tol = 1e-11 if dt == torch.float64 else _scan_f32_tol(3, L)
    for left in (True, False):
        y = torch.ops.b200pose.cumprod(xd, grp, left).double().cpu().numpy()
        ref = S.cumprod(grp, xd.double().cpu().numpy(), left)
        _within(f"cumprod {grp} {dt} B=3 L={L} left={left}", np.abs(y - ref).max(), 1 + np.abs(ref).max(), tol)


@pytest.mark.gpu
def test_imu_module_gpu(golden_scan):
    _check_imu_module(golden_scan, "cuda", 1e-10)


@pytest.mark.gpu
@pytest.mark.parametrize("dt_", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("B,F", [(3, 2), (5, 254), (4, 256), (7, 258), (2, 1000), (3, 10_000), (2, 777)])
def test_imu_tma_staged_kernel_matches_register_kernel(dt_, B, F):
    """csrc/scan.cu imu_predict_tma_kernel (samples through a TMA-fed shared-memory ring, bulk stores) against
    imu_integrate_kernel: same arithmetic in the same order, so the outputs are compared bit for bit; lengths below, at and
    above the tile, several tiles, with initial states; F = 777 (rows not 16-byte multiples) must fall back and still agree.
    The fp64 result is also checked against the oracle."""
    import ctypes
    from pypose_b200 import _C
    torch.manual_seed(F + B)
    dt = (0.004 + 0.002 * torch.rand(B, F, 1, dtype=dt_, device="cuda"))
    gyro = 0.3 * torch.randn(B, F, 3, dtype=dt_, device="cuda")
    acc = torch.randn(B, F, 3, dtype=dt_, device="cuda") + torch.tensor([0, 0, 9.81], dtype=dt_, device="cuda")
    init = {"pos": torch.randn(B, 1, 3, dtype=dt_, device="cuda"), "rot": pp.randn_SO3(B, 1, dtype=dt_, device="cuda"),
            "vel": torch.randn(B, 1, 3, dtype=dt_, device="cuda")}
    mode = _C.lib().b200_imu_tma_mode
    mode.restype, mode.argtypes = ctypes.c_int, [ctypes.c_int]
    prev = mode(-1)
    outs = {}
    try:
        for m in (0, 1):
            mode(m)
            imu = pp.module.IMUPreintegrator(prop_cov=False, reset=True).to(dt_).cuda()
            o = imu(dt, gyro, acc, init_state=init)
            outs[m] = {k: (o[k].tensor() if hasattr(o[k], "tensor") else o[k]).clone() for k in ("rot", "vel", "pos")}
    finally:
        mode(prev)
    for k in ("rot", "vel", "pos"):
        assert torch.isfinite(outs[1][k]).all()
        assert torch.equal(outs[0][k], outs[1][k]), (k, (outs[0][k] - outs[1][k]).abs().max().item())
    if dt_ == torch.float64:
        o = S.imu_integrate(dt.cpu().numpy(), gyro.cpu().numpy(), acc.cpu().numpy(), init_rot=init["rot"].tensor().cpu().numpy())
        Dp, Dv, Dr, Dt = o[1], o[2], o[3], o[4]
        R0 = init["rot"].tensor().cpu().numpy().reshape(B, 1, 4).repeat(F, 1).reshape(-1, 4)
        rot_ref = O.mul("SO3", R0, Dr.reshape(-1, 4))
        d = O.log("SO3", O.mul("SO3", O.inv("SO3", rot_ref), outs[1]["rot"].cpu().numpy().reshape(-1, 4)))
        assert np.abs(d).max() <= 1e-10
        v0 = init["vel"].cpu().numpy()
        vel_ref = v0 + O.act("SO3", R0, Dv.reshape(-1, 3)).reshape(B, F, 3)
        assert np.abs(outs[1]["vel"].cpu().numpy() - vel_ref).max() <= 1e-10 * (1 + np.abs(vel_ref).max())


@pytest.mark.gpu
def test_imu_config4_size_vs_oracle_subset():
    """BASELINE.json configs[3]: 1e3 trajectories x 1e4 samples, fp64; the first 4 trajectories are
    checked against the oracle (rot via Log(a^-1 b) <= 1e-9, vel/pos relative 1e-9, SURVEY.md §8d)."""
    torch.manual_seed(0)
    B, F = 1000, 10_000
    dt = torch.full((B, F, 1), 0.005, dtype=torch.float64, device="cuda")
    gyro = 0.1 * torch.randn(B, F, 3, dtype=torch.float64, device="cuda")
    acc = torch.randn(B, F, 3, dtype=torch.float64, device="cuda") + torch.tensor([0, 0, 9.81], dtype=torch.float64, device="cuda")
    m = pp.module.IMUPreintegrator(prop_cov=False, reset=True).double().cuda()
    out = m(dt, gyro, acc)
    o = S.imu_integrate(dt[:4].cpu().numpy(), gyro[:4].cpu().numpy(), acc[:4].cpu().numpy())
    Dp, Dv, Dr = o[1], o[2], o[3]
    # default init state is identity / zeros -> predict == integrate
    rot = out["rot"].tensor()[:4].cpu().numpy()
    d = O.log("SO3", O.mul("SO3", O.inv("SO3", Dr.reshape(-1, 4)), rot.reshape(-1, 4)))
    assert np.abs(d).max() <= 1e-9
    assert np.abs(out["vel"][:4].cpu().numpy() - Dv).max() <= 1e-9 * (1 + np.abs(Dv).max())
    assert np.abs(out["pos"][:4].cpu().numpy() - Dp).max() <= 1e-9 * (1 + np.abs(Dp).max())
    assert torch.isfinite(out["pos"]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 5, 127, 128, 129, 1000])
def test_imu_cov_kernel_vs_oracle(F):
    from tests.util import rand_group
    rng = np.random.default_rng(F)
    B = 5
    Rk = rand_group(rng, "SO3", B * F, tmax=0.05).reshape(B, F, 4)
    Rij = rand_group(rng, "SO3", B * F, tmax=2.0).reshape(B, F, 4)
    a = rng.standard_normal((B, F, 3)) * 3
    dt = 0.005 * (1 + 0.2 * rng.random((B, F, 1)))
    gc, ac = np.abs(rng.standard_normal((B, 1, 3))) * 1e-4, np.abs(rng.standard_normal((B, 1, 3))) * 1e-2
    A0 = rng.standard_normal((B, 9, 9)) * 1e-3
    init = A0 @ np.swapaxes(A0, -1, -2)
    c = lambda x: torch.from_numpy(x).cuda()
    cov = torch.ops.b200pose.imu_cov(c(Rk), c(Rij), c(a), c(dt), c(gc), c(ac), c(init)).cpu().numpy()
    ref = S.imu_cov(Rk, Rij, a, dt, gc, ac, init)
    assert np.abs(cov - ref).max() <= 1e-11 * max(1.0, np.abs(ref).max()), np.abs(cov - ref).max()
    # per-sample covariances
    gcf, acf = np.abs(rng.standard_normal((B, F, 3))) * 1e-4, np.abs(rng.standard_normal((B, F, 3))) * 1e-2
    cov = torch.ops.b200pose.imu_cov(c(Rk), c(Rij), c(a), c(dt), c(gcf), c(acf), c(init[:1])).cpu().numpy()
    ref = S.imu_cov(Rk, Rij, a, dt, gcf, acf, init[:1])
    assert np.abs(cov - ref).max() <= 1e-11 * max(1.0, np.abs(ref).max())


@pytest.mark.gpu
def test_imu_config4_with_covariance_runs_at_full_size():
    """BASELINE.json configs[3], second run: prop_cov=True at B=1e3, F=1e4 fp64 (the reference needs 6.5 GB for A alone
    and was measured at B <= 100, SURVEY.md §6); covariance symmetric PSD-ish and finite; first trajectories vs oracle."""
    torch.manual_seed(1)
    B, F = 1000, 10_000
    dt = torch.full((B, F, 1), 0.005, dtype=torch.float64, device="cuda")
    gyro = 0.1 * torch.randn(B, F, 3, dtype=torch.float64, device="cuda")
    acc = torch.randn(B, F, 3, dtype=torch.float64, device="cuda") + torch.tensor([0, 0, 9.81], dtype=torch.float64, device="cuda")
    m = pp.module.IMUPreintegrator(prop_cov=True, reset=True).double().cuda()
    out = m(dt, gyro, acc)
    cov = out["cov"]
    assert cov.shape == (B, 9, 9) and torch.isfinite(cov).all()
    assert (cov - cov.mT).abs().max() <= 1e-9 * cov.abs().max()
    inte = S.imu_integrate(dt[:2].cpu().numpy(), gyro[:2].cpu().numpy(), acc[:2].cpu().numpy())
    a_, Dr, w = inte[0], inte[3], inte[5]
    gcv = np.full((2, 1, 3), (3.2e-3) ** 2)
    acv = np.full((2, 1, 3), (8e-2) ** 2)
    ref = S.imu_cov(w, Dr, a_, dt[:2].cpu().numpy(), gcv.astype(np.float32).astype(np.float64), acv.astype(np.float32).astype(np.float64),
                    np.zeros((1, 9, 9)))
    assert np.abs(cov[:2].cpu().numpy() - ref).max() <= 1e-8 * np.abs(ref).max()


def _check_imu_gradients(dev, tol):
    """ADVICE r1: the integrator is differentiable in the signals and the initial state like the reference
    (goldens: oracle/make_golden_imu_grad.py, reference fp64)."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "scan_imu.npz"))
    gg = np.load(os.path.join(os.path.dirname(__file__), "golden", "imu_grad.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    for tag in ("free", "rot"):
        for cov in (False, True):
            dt, gyro, acc = (t(k).requires_grad_() for k in ("imu/dt", "imu/gyro", "imu/acc"))
            pos, vel = t("imu/init_pos").requires_grad_(), t("imu/init_vel").requires_grad_()
            init = {"pos": pos, "rot": pp.SO3(t("imu/init_rot")), "vel": vel}
            kw = {"rot": pp.SO3(t("imu/rot"))} if tag == "rot" else {}
            m = pp.module.IMUPreintegrator(prop_cov=cov, reset=True).double().to(dev)
            out = m(dt, gyro, acc, init_state=init, **kw)
            s = (out["pos"] ** 2).sum() + (out["vel"] ** 2).sum() + (out["rot"].Log().tensor() ** 2).sum()
            s.backward()
            key = f"{tag}/{'cov' if cov else 'nocov'}"
            np.testing.assert_allclose(float(s), gg[f"{key}/scalar"], rtol=tol)
            for name, v in (("dt", dt), ("gyro", gyro), ("acc", acc), ("pos", pos), ("vel", vel)):
                ref = gg[f"{key}/grad_{name}"]
                np.testing.assert_allclose(v.grad.cpu().numpy(), ref, atol=tol * (1 + np.abs(ref).max()), err_msg=f"{key}/{name}")
            # integrate() alone is differentiable too
            d = m.integrate(dt, gyro, acc, init_rot=init["rot"], **kw)
            assert d["Dp"].requires_grad and d["Dr"].requires_grad


def test_imu_gradients_cpu():
    _check_imu_gradients("cpu", 1e-9)


@pytest.mark.gpu
def test_imu_gradients_gpu():
    _check_imu_gradients("cuda", 1e-9)


def test_imu_gravity_buffer_is_honoured():
    m = pp.module.IMUPreintegrator(prop_cov=False, reset=True).double()
    dt = torch.full((1, 5, 1), 0.01, dtype=torch.float64)
    z = torch.zeros(1, 5, 3, dtype=torch.float64)
    a = m(dt, z, z)["vel"][0, -1]
    m.gravity = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    b = m(dt, z, z)["vel"][0, -1]
    assert abs(float(a[2]) + 0.05 * 9.81007) < 1e-6 and abs(float(b[2]) + 0.05) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("grp", GROUPS)
@pytest.mark.parametrize("B,L", [(1, 1_000_000), (3, 40_000), (2, 4097), (1, 1_200_000)])
def test_cumprod_time_split_lookback_vs_oracle(grp, B, L):
    """VERDICT r1 item 7: (B = 1, L = 1e6) used to run on one SM.  The time-split kernels (tile products, scan of the tile
    products, apply; csrc/scan.cu cumprod_tile_*, taken while B < 2 SMs and L >= 4 tiles) against the log-step reference
    (_scan_logstep), both directions, fp64 at 1e-11 and fp32 at _scan_f32_tol; two runs are bit-identical in each dtype.
    At L = 4097 the log-step reference is itself checked against the sequential oracle.  cumprod_tile_prefix_kernel
    carries across its 1024-tile rounds from L > 524,288 in fp64 (L = 1e6: 1954 tiles) and L > 1,048,576 in fp32
    (L = 1.2e6: 1172 tiles); those two lengths run in the dtype whose rounds they cross, the others in both.  Each dtype
    is compared with the reference evaluated on its own rows upcast to fp64 (fp32-rounded quaternions are not unit, and
    the translation groups' product is associative only for unit quaternions)."""
    from tests.util import rand_group
    rng = np.random.default_rng(L + B)
    x = rand_group(rng, grp, B * L, tmin=0.0, tmax=0.02, t_sigma=0.01, s_sigma=1e-5).reshape(B, L, -1)
    dts = {1_000_000: (torch.float64,), 1_200_000: (torch.float32,)}.get(L, (torch.float64, torch.float32))
    for dt in dts:
        xt = torch.from_numpy(x).to(dt).cuda()
        xh = xt.double().cpu().numpy()
        for left in (True, False):
            ref = _scan_logstep(grp, xh, left)
            if L <= 4097 and dt == torch.float64:
                seq = S.cumprod(grp, xh, left)
                assert np.abs(ref - seq).max() <= 1e-12 * (1 + np.abs(seq).max()), (grp, left)
            y = torch.ops.b200pose.cumprod(xt, grp, left)
            assert torch.equal(y, torch.ops.b200pose.cumprod(xt, grp, left))
            tol = 1e-11 if dt == torch.float64 else _scan_f32_tol(B, L)
            _within(f"cumprod time-split {grp} {dt} B={B} L={L} left={left}", np.abs(y.double().cpu().numpy() - ref).max(),
                    1 + np.abs(ref).max(), tol)


def test_scan_logstep_matches_sequential_oracle():
    """The log-step reference used at long lengths agrees with the sequential oracle (every group, both directions,
    lengths at and around powers of two)."""
    from tests.util import rand_group
    rng = np.random.default_rng(5)
    for grp in GROUPS:
        for L in (1, 2, 3, 64, 65, 300):
            x = rand_group(rng, grp, 2 * L, tmax=0.5, t_sigma=0.3, s_sigma=0.05).reshape(2, L, -1)
            for left in (True, False):
                seq = S.cumprod(grp, x, left)
                assert np.abs(_scan_logstep(grp, x, left) - seq).max() <= 1e-13 * (1 + np.abs(seq).max()), (grp, L, left)


@pytest.mark.gpu
@pytest.mark.parametrize("grp", GROUPS)
@pytest.mark.parametrize("L", [1025, 3000])
def test_cumprod_single_pass_many_tiles_large_batch(grp, L):
    """cumprod_kernel over several tiles (fp32: 2-3 tiles of 1024 rows, fp64: 3-6 tiles of 512) with B = 2 SMs + 1
    sequences, which _cumprod_cuda keeps on the single-pass kernel (the time-split route needs B < 2 SMs), both dtypes
    and directions against the log-step reference on each dtype's rows; fp64 1e-11, fp32 _scan_f32_tol."""
    from tests.util import rand_group
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    rng = np.random.default_rng(L)
    x = rand_group(rng, grp, B * L, tmax=0.3, t_sigma=0.1, s_sigma=0.02).reshape(B, L, -1)
    for dt in (torch.float64, torch.float32):
        xt = torch.from_numpy(x).to(dt).cuda()
        xh = xt.double().cpu().numpy()
        for left in (True, False):
            ref = _scan_logstep(grp, xh, left)
            y = torch.ops.b200pose.cumprod(xt, grp, left).double().cpu().numpy()
            tol = 1e-11 if dt == torch.float64 else _scan_f32_tol(B, L)
            _within(f"cumprod single-pass {grp} {dt} B={B} L={L} left={left}", np.abs(y - ref).max(), 1 + np.abs(ref).max(), tol)


@pytest.mark.gpu
@pytest.mark.parametrize("grp", ["SE3", "Sim3"])
@pytest.mark.parametrize("dt", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("B,L", [(4, 1000), (1, 5000)], ids=["single", "split"])
def test_cumprod_misaligned_base_is_bitwise_aligned(grp, dt, B, L):
    """An input whose base pointer is one element past a 16-byte boundary (a contiguous view at storage offset 1) is
    staged by the scalar branch of tile_load; with 7 / 8 words per row every tile of an aligned input takes the vector
    branch instead.  Both routes (single pass: B = 4, L = 1000; time split: B = 1, L = 5000): the result is bitwise
    equal to the same rows at an aligned address."""
    from tests.util import rand_group
    rng = np.random.default_rng(B * L)
    x = torch.from_numpy(rand_group(rng, grp, B * L, tmax=0.3, t_sigma=0.1, s_sigma=0.02).reshape(B, L, -1)).to(dt).cuda()
    buf = torch.empty(x.numel() + 1, dtype=dt, device="cuda")
    xm = buf[1:].view(x.shape)
    xm.copy_(x)
    assert xm.is_contiguous() and xm.data_ptr() % 16 != 0 and x.data_ptr() % 16 == 0
    for left in (True, False):
        assert torch.equal(torch.ops.b200pose.cumprod(xm, grp, left), torch.ops.b200pose.cumprod(x, grp, left)), left


# ------------------------------------------------------------------ IMU routes vs the oracle
IMU_F = [1, 127, 128, 129, 255, 256, 257, 1000, 10_000]
IMU_CASES = ["per_traj", "bcast", "mixed", "rot_seq", "rot_b1", "gravity", "big_rot"]


def _imu_tol(dtype, F):
    """(rotation angle, relative) bounds of the IMU outputs.  fp64: the 1e-10 of the module tests.  fp32: unit roundoff
    times the samples a prefix runs over plus the in-tile shuffle depth (the rotation and (v, p, t) scans add one
    rounding per sample); the vectors also integrate the rotation's error against gravity, hence twice that.  Measured
    on an H100 up to F = 1e4 (DESIGN.md §4): 0.25 and 0.5 of these bounds."""
    if dtype == torch.float64:
        return 1e-10, 1e-10
    return U32 * (F + 16), 2 * U32 * (F + 16)


def _imu_inputs(case, B, F, dtype, seed):
    rng = np.random.default_rng(seed)
    dt = 0.005 * (1 + 0.2 * rng.random((B, F, 1)))
    gyro = 0.3 * rng.standard_normal((B, F, 3))
    acc = rng.standard_normal((B, F, 3)) + np.array([0, 0, 9.81])
    if case == "big_rot":
        # every 37th sample turns by 0.2 .. 3 rad, every 53rd (from the 5th) has gyro exactly zero, one turns by pi - 5e-4:
        # warps of imu_integrate_kernel / imu_predict_tma_kernel that mix both branches of so3_exp_imu
        ax = rng.standard_normal((B, F, 3))
        ax /= np.linalg.norm(ax, axis=-1, keepdims=True)
        big = np.arange(F) % 37 == 0
        gyro[:, big] = ax[:, big] * rng.uniform(0.2, 3.0, (B, int(big.sum()), 1)) / dt[:, big]
        gyro[:, np.arange(F) % 53 == 5] = 0.0
        gyro[:, F // 2] = ax[:, F // 2] * (np.pi - 5e-4) / dt[:, F // 2]
    from tests.util import rand_group
    nb = lambda which: B if which else 1
    init_rot = rand_group(rng, "SO3", nb(case != "bcast" and case != "mixed")).reshape(-1, 1, 4)
    init_pos = rng.standard_normal((nb(case not in ("bcast", "mixed")), 1, 3))
    init_vel = rng.standard_normal((nb(case != "bcast"), 1, 3))
    rot = None
    if case == "rot_seq":
        rot = rand_group(rng, "SO3", B * F, tmax=1.0).reshape(B, F, 4)
    elif case == "rot_b1":
        rot = rand_group(rng, "SO3", B, tmax=1.0).reshape(B, 1, 4)
    gravity = [0.0, 0.0, float(np.float32(9.81007))]
    if case == "gravity":
        gravity = [0.375, -1.25, 9.5]                  # exact in fp32: the kernel and the oracle see the same vector
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()
    return {k: t(v) for k, v in (("dt", dt), ("gyro", gyro), ("acc", acc), ("rot", rot), ("init_rot", init_rot),
                                 ("init_pos", init_pos), ("init_vel", init_vel))}, gravity


def _imu_reference(inp, gravity):
    """fp64 oracle of every output the IMU routes write, on the fp64 upcast of the kernel's inputs."""
    n = {k: None if v is None else v.double().cpu().numpy() for k, v in inp.items()}
    B, F = n["dt"].shape[:2]
    rot = None if n["rot"] is None else np.broadcast_to(n["rot"], (B, F, 4))
    a, Dp, Dv, Dr, Dt, w = S.imu_integrate(n["dt"], n["gyro"], n["acc"], rot, n["init_rot"], gravity)
    R0 = np.broadcast_to(n["init_rot"], (B, F, 4)).reshape(-1, 4)
    p0, v0 = n["init_pos"], n["init_vel"]
    return {"a": a, "Dp": Dp, "Dv": Dv, "Dr": Dr, "Dt": Dt, "w": w,
            "rot": O.mul("SO3", R0, Dr.reshape(-1, 4)).reshape(B, F, 4),
            "vel": v0 + O.act("SO3", R0, Dv.reshape(-1, 3)).reshape(B, F, 3),
            "pos": p0 + O.act("SO3", R0, Dp.reshape(-1, 3)).reshape(B, F, 3) + v0 * Dt}


def _check_imu_outputs(route, got, ref, tol_rot, tol_rel):
    for k, v in got.items():
        v = v.double().cpu().numpy()
        r = ref[k]
        assert np.isfinite(v).all(), (route, k)
        if k in ("Dr", "w", "rot"):
            d = O.log("SO3", O.mul("SO3", O.inv("SO3", r.reshape(-1, 4)), v.reshape(-1, 4)))
            _within(f"imu {route} {k}", np.linalg.norm(d, axis=-1).max(), 1.0, tol_rot)
        else:
            _within(f"imu {route} {k}", np.abs(v - r).max(), 1 + np.abs(r).max(), tol_rel)


@pytest.mark.gpu
@pytest.mark.parametrize("case", IMU_CASES)
@pytest.mark.parametrize("F", IMU_F)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
def test_imu_every_route_vs_oracle(dtype, F, case):
    """Every route of b200_imu_integrate_{f32,f64} against the fp64 oracle, each output it writes:
      tma        imu_predict, b200_imu_tma_mode 1: imu_predict_tma_kernel when nothing but rot/vel/pos is written, no
                 known rot and every array 16-byte aligned with F * sizeof a multiple of 16 (fp32: F % 4 == 0, fp64:
                 F % 2 == 0), imu_integrate_kernel otherwise;
      register   imu_predict, mode 0: imu_integrate_kernel (CH = 2, 256-sample tiles), predicted states only;
      full       imu_full (prop_cov=True forward): imu_integrate_kernel with a_out set (fp64 CH = 1, 128-sample tiles;
                 fp32 CH = 2), all nine outputs;
      integrate  imu_integrate with init_rot: the six increments.
    F puts every kernel below, at and above its tile and up to 10 000 samples (40-80 tiles); initial states per
    trajectory, batch-1 broadcast and mixed (pos batch 1, vel batch B); known rotations per sample and (B, 1, 4);
    a non-default gravity; large rotations that take the general branch of so3_exp_imu in some lanes of a warp."""
    import ctypes
    from pypose_b200 import _C
    B = 3
    inp, grav = _imu_inputs(case, B, F, dtype, seed=F * 10 + IMU_CASES.index(case))
    ref = _imu_reference(inp, grav)
    tol_rot, tol_rel = _imu_tol(dtype, F)
    ops = torch.ops.b200pose
    pred = (inp["dt"], inp["gyro"], inp["acc"], inp["rot"], inp["init_rot"], inp["init_pos"], inp["init_vel"], grav)
    mode = _C.lib().b200_imu_tma_mode
    mode.restype, mode.argtypes = ctypes.c_int, [ctypes.c_int]
    prev = mode(-1)
    try:
        for m, route in ((1, "tma"), (0, "register")):
            mode(m)
            r, v, p = ops.imu_predict(*pred)
            _check_imu_outputs(f"{route} {dtype} F={F} {case}", {"rot": r, "vel": v, "pos": p}, ref, tol_rot, tol_rel)
    finally:
        mode(prev)
    full = ops.imu_full(*pred)
    names = ("a", "Dp", "Dv", "Dr", "Dt", "w", "rot", "vel", "pos")
    _check_imu_outputs(f"full {dtype} F={F} {case}", dict(zip(names, full)), ref, tol_rot, tol_rel)
    init_t = inp["init_rot"] if inp["rot"] is None else None
    inte = ops.imu_integrate(inp["dt"], inp["gyro"], inp["acc"], inp["rot"], init_t, grav)
    _check_imu_outputs(f"integrate {dtype} F={F} {case}", dict(zip(names[:6], inte)), ref, tol_rot, tol_rel)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("F", [256, 1000])
def test_imu_misaligned_inputs_fall_back_bitwise(dtype, F):
    """dt / gyro / acc at storage offset 1 fail the 16-byte test of IMU_ABI, so the predict call that took
    imu_predict_tma_kernel falls back to imu_integrate_kernel: the result is bitwise equal to the aligned call (same
    arithmetic in the same order); the full route on the same inputs is bitwise equal too."""
    inp, grav = _imu_inputs("per_traj", 3, F, dtype, seed=F)

    def shifted(t):
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.is_contiguous() and v.data_ptr() % 16 != 0
        return v

    mis = dict(inp, dt=shifted(inp["dt"]), gyro=shifted(inp["gyro"]), acc=shifted(inp["acc"]))
    args = lambda d: (d["dt"], d["gyro"], d["acc"], None, d["init_rot"], d["init_pos"], d["init_vel"], grav)
    for op in (torch.ops.b200pose.imu_predict, torch.ops.b200pose.imu_full):
        for x, y in zip(op(*args(inp)), op(*args(mis))):
            assert torch.equal(x, y), op


# ------------------------------------------------------------------ covariance chunking
IMU_COV_CHUNKS = [(1, 300, 1), (2, 300, 300), (3, 300, 512), (4, 320, 10), (5, 330, 10), (6, 640, 10), (7, 650, 10),
                  (8, 1000, 10), (9, 1000, 7)]


def _imu_cov_inputs(rng, B, F, per_sample, init_per_traj):
    from tests.util import rand_group
    Rk = rand_group(rng, "SO3", B * F, tmax=0.05).reshape(B, F, 4)
    Rij = rand_group(rng, "SO3", B * F, tmax=2.0).reshape(B, F, 4)
    a = rng.standard_normal((B, F, 3)) * 3
    dt = 0.005 * (1 + 0.2 * rng.random((B, F, 1)))
    nf = F if per_sample else 1
    gc, ac = np.abs(rng.standard_normal((B, nf, 3))) * 1e-4, np.abs(rng.standard_normal((B, nf, 3))) * 1e-2
    A0 = rng.standard_normal((B if init_per_traj else 1, 9, 9)) * 1e-3
    return Rk, Rij, a, dt, gc, ac, A0 @ np.swapaxes(A0, -1, -2)


def _cov_f32_tol(F, chunk):
    """fp32 bound of the covariance relative to max|truth|: unit roundoff times the sequential steps behind an entry
    (chunk steps in imu_cov_chunk_prod_kernel / imu_cov_accum_kernel, NC steps of the suffix scan, NC partial sums in
    imu_cov_finish_kernel) plus the 16 terms of a 9x9 entry.  Measured on an H100 (DESIGN.md §4): <= 0.07 of it."""
    NC = -(-F // chunk)
    return U32 * (min(chunk, F) + 2 * NC + 16)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("noise", ["traj_noise_shared_init", "sample_noise_traj_init", "traj_noise_traj_init",
                                   "sample_noise_shared_init"])
@pytest.mark.parametrize("case", [c[0] for c in IMU_COV_CHUNKS])
def test_imu_cov_chunking_vs_oracle(case, noise, dtype):
    """imu_cov_chunk_prod / suffix / accum / finish through _imu_cov_cuda with an explicit chunk (the op schema has none,
    and the default min(256, max(16, B F / 65536)) is 16 at these sizes): chunk = 1 (NC = F), chunk >= F (NC = 1),
    NC = 32, 33, 64, 65, 100 (one, two and more 32-chunk rounds of imu_cov_suffix_kernel) and a chunk that does not divide
    F; noise per trajectory or per sample, init_cov shared or per trajectory.  fp64 at 1e-11 of max|truth| as the
    module tests, fp32 at _cov_f32_tol."""
    from pypose_b200.lietensor.scan import _imu_cov_cuda
    _, F, chunk = IMU_COV_CHUNKS[case - 1]
    rng = np.random.default_rng(case * 7 + len(noise))
    B = 5
    ins = _imu_cov_inputs(rng, B, F, noise.startswith("sample"), noise.endswith("traj_init"))
    c = lambda x: torch.from_numpy(x).to(dtype).cuda()
    ins_t = [c(x) for x in ins]
    cov = _imu_cov_cuda(*ins_t, chunk=chunk).double().cpu().numpy()
    ref = S.imu_cov(*[t.double().cpu().numpy() for t in ins_t])
    tol = 1e-11 if dtype == torch.float64 else _cov_f32_tol(F, chunk)
    _within(f"imu_cov {dtype} F={F} chunk={chunk} {noise}", np.abs(cov - ref).max(), np.abs(ref).max(), tol)


# ------------------------------------------------------------------ streaming preintegration (reset=False)
def _imu_stream_golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "imu_stream.npz"))


def _check_imu_stream(dev):
    """The default IMUPreintegrator (reset=False, prop_cov=True) over three consecutive windows of 50, 1 and 77 samples,
    the second with its own gyro_cov / acc_cov, free and with known rotations: every window's rot / vel / pos / cov and
    the state carried to the next call (pos, rot, vel, cov, Rij) reproduce the reference (oracle/make_golden_imu_stream.py)
    to 1e-10 of each array's scale."""
    g = _imu_stream_golden()
    for tag in ("free", "rot"):
        m = pp.module.IMUPreintegrator().double().to(dev)
        w = 0
        while f"in/{w}/dt" in g.files:
            t = lambda k: torch.from_numpy(g[f"in/{w}/{k}"]).to(dev)
            kw = {"rot": pp.SO3(t("rot"))} if tag == "rot" else {}
            if f"in/{w}/gyro_cov" in g.files:
                kw.update(gyro_cov=t("gyro_cov"), acc_cov=t("acc_cov"))
            out = m(t("dt"), t("gyro"), t("acc"), **kw)
            got = {f"out/{k}": out[k] for k in ("pos", "vel", "rot", "cov")}
            got.update({f"state/{k}": getattr(m, k) for k in ("pos", "rot", "vel", "cov", "Rij")})
            for k, v in got.items():
                v = (v.tensor() if isinstance(v, pp.LieTensor) else v).cpu().numpy()
                ref = g[f"{tag}/{w}/{k}"]
                assert v.shape == ref.shape, (tag, w, k)
                _within(f"stream {tag} window {w} {k}", np.abs(v - ref).max(), np.abs(ref).max(), 1e-10)
            w += 1
        assert w == 3


def test_imu_stream_reset_false_cpu():
    _check_imu_stream("cpu")


@pytest.mark.gpu
def test_imu_stream_reset_false_gpu():
    """The fused route (imu_full + imu_cov) of the default, state-carrying IMUPreintegrator."""
    _check_imu_stream("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
def test_imu_stream_long_windows_vs_chained_oracle(dtype):
    """reset=False over windows of 1000, 1 and 5000 samples (imu_integrate_kernel over 8-40 tiles, the covariance with
    the default chunking) against S.imu_integrate / S.imu_cov chained by hand: each window starts from the previous
    one's last pos / rot / vel, its covariance and Rij = Rij_prev * Dr."""
    B = 2
    rng = np.random.default_rng(17)
    m = pp.module.IMUPreintegrator().to(dtype).cuda()
    gc = np.broadcast_to(m.gyro_cov.double().cpu().numpy(), (B, 1, 3))
    ac = np.broadcast_to(m.acc_cov.double().cpu().numpy(), (B, 1, 3))
    grav = [0.0, 0.0, m._g]
    p, R, v = np.zeros((1, 1, 3)), np.array([[[0.0, 0, 0, 1]]]), np.zeros((1, 1, 3))
    cov, Rij = np.zeros((1, 9, 9)), None
    tol_rot, tol_rel = _imu_tol(dtype, 6001)
    tol_cov = 1e-10 if dtype == torch.float64 else _cov_f32_tol(5000, 16)
    for w, F in enumerate((1000, 1, 5000)):
        dt = torch.from_numpy(0.005 * (1 + 0.2 * rng.random((B, F, 1)))).to(dtype)
        gyro = torch.from_numpy(0.3 * rng.standard_normal((B, F, 3))).to(dtype)
        acc = torch.from_numpy(rng.standard_normal((B, F, 3)) + np.array([0, 0, 9.81])).to(dtype)
        out = m(dt.cuda(), gyro.cuda(), acc.cuda())
        n = lambda x: x.double().numpy()
        a, Dp, Dv, Dr, Dt, wq = S.imu_integrate(n(dt), n(gyro), n(acc), None, R, grav)
        R0 = np.broadcast_to(R, (B, F, 4)).reshape(-1, 4)
        ref = {"rot": O.mul("SO3", R0, Dr.reshape(-1, 4)).reshape(B, F, 4),
               "vel": v + O.act("SO3", R0, Dv.reshape(-1, 3)).reshape(B, F, 3)}
        ref["pos"] = p + O.act("SO3", R0, Dp.reshape(-1, 3)).reshape(B, F, 3) + v * Dt
        Rseq = Dr if Rij is None else O.mul("SO3", np.broadcast_to(Rij, (B, F, 4)).reshape(-1, 4), Dr.reshape(-1, 4)).reshape(B, F, 4)
        cov = S.imu_cov(wq, Rseq, a, n(dt), gc, ac, cov)
        _check_imu_outputs(f"stream {dtype} window {w}", {k: out[k].tensor() if k == "rot" else out[k] for k in ref}, ref,
                           tol_rot, tol_rel)
        _within(f"stream {dtype} window {w} cov", np.abs(out["cov"].double().cpu().numpy() - cov).max(), np.abs(cov).max(),
                tol_cov)
        p, R, v, Rij = ref["pos"][:, -1:], ref["rot"][:, -1:], ref["vel"][:, -1:], Rseq[:, -1:]
