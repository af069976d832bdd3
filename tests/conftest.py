"""pytest configuration.

* registers the `gpu` marker (tests that need a real H100);
* gives the `b200pose::*` torch ops a **test-only CPU kernel backed by the oracle**, so the
  host-side logic (LieTensor dispatch, autograd/vmap registrations, LM control flow, gloo
  sharding) can be exercised without a GPU.  The shipped package registers CUDA kernels only —
  without this conftest a CPU tensor raises in the dispatcher (tests/test_abi.py checks that in a
  clean subprocess).
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def _install_cpu_oracle_kernels():
    import pypose_b200  # noqa: F401  (defines the ops)
    from pypose_b200.lietensor import ops as _ops
    from oracle import lie_oracle

    def make(name):
        sym = name

        def cpu_impl(*ts):
            arrs = [t.detach().contiguous().numpy() for t in ts]
            outs = lie_oracle.run(sym, *arrs)
            outs = [torch.from_numpy(np.ascontiguousarray(o)).to(ts[0].dtype) for o in outs]
            return outs[0] if len(outs) == 1 else tuple(outs)
        return cpu_impl

    for name in _ops.OP_INFO:
        torch.library.impl(f"b200pose::{name}", "CPU")(make(name))
    try:
        from pypose_b200 import _testhooks
        _testhooks.install_cpu_oracle()
    except ImportError:
        pass


_install_cpu_oracle_kernels()


@pytest.fixture(scope="session")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "lie_ops.npz"))


def _install_cpu_oracle_lm_kernels():
    """Test-only CPU kernels for the fused LM ops, backed by oracle/lm_oracle.py."""
    from pypose_b200.optim import _fused  # noqa: F401
    from oracle import lm_oracle as L

    def t(a, like):
        return torch.from_numpy(np.ascontiguousarray(a)).to(like.dtype)

    def f64(a):
        return torch.from_numpy(np.asarray(a, dtype=np.float64))

    def n(x):
        return x.detach().double().numpy()

    def poseinv_loss(P, X, robust, delta):
        return f64(L.poseinv_loss(n(P), n(X), robust, delta))

    def poseinv_trial(P, X, scale, dmin, dmax, robust, delta):
        Pt, sums = L.poseinv_trial(n(P), n(X), scale, dmin, dmax, robust, delta)
        return t(Pt, P), f64(sums)

    def reproj_accum(poses, pts, pix, seg, robust, delta):
        H, g, s = L.reproj_accum(n(poses), n(pts), n(pix), seg.numpy(), robust, delta)
        return t(H, poses), t(g, poses), f64(s)

    def solve6_retract(H, g, P, scale, dmin, dmax):
        Pt, D, s = L.solve6_retract(n(H), n(g), n(P), scale, dmin, dmax)
        return t(Pt, P), t(D, P), f64(s)

    def reproj_loss(poses, pts, pix, seg, robust, delta):
        cidx = np.repeat(np.arange(poses.shape[0]), np.diff(seg.numpy()))
        return f64(L.reproj_loss(n(poses), n(pts), n(pix), cidx, robust, delta))

    def reproj_residual(poses, pts, pix, cidx):
        return t(L.reproj_residual(n(poses), n(pts), n(pix), cidx.numpy()), poses)

    def pgo_linearize(nodes, Z, ei, ej, robust, delta):
        M, u, c = L.pgo_linearize(n(nodes), n(Z), ei.numpy(), ej.numpy(), robust, delta)
        return t(M, nodes), t(u, nodes), f64(c)

    def pgo_linearize_w(nodes, Z, ei, ej, W, robust, delta):
        outs = L.pgo_linearize(n(nodes), n(Z), ei.numpy(), ej.numpy(), robust, delta, W=n(W))
        return (*[t(o, nodes) for o in outs[:4]], f64(outs[4]))

    def pgo_scatter(M, u, ei, ej, nn):
        Hd, g = L.pgo_scatter(n(M), n(u), ei.numpy(), ej.numpy(), nn)
        return t(Hd, M), t(g, M)

    def pgo_spmv(M, ei, ej, x, y0):
        return t(L.pgo_spmv(n(M), ei.numpy(), ej.numpy(), n(x), n(y0)), M)

    def pgo_loss(nodes, Z, ei, ej, robust, delta):
        return f64(L.pgo_loss(n(nodes), n(Z), ei.numpy(), ej.numpy(), robust, delta))

    def ba_linearize(poses, points, pix, cidx, pidx, robust, delta):
        outs = L.ba_linearize(n(poses), n(points), n(pix), cidx.numpy(), pidx.numpy(), robust, delta)
        return tuple(t(o, poses) for o in outs[:7]) + (f64(outs[7]),)

    def ba_wtx(Jc, Jp, cidx, pidx, x, npts):
        return t(L.ba_wtx(n(Jc), n(Jp), cidx.numpy(), pidx.numpy(), n(x), npts), Jc)

    def ba_wv(Jc, Jp, cidx, pidx, v, ncam):
        return t(L.ba_wv(n(Jc), n(Jp), cidx.numpy(), pidx.numpy(), n(v), ncam), Jc)

    def ba_loss(poses, points, pix, cidx, pidx, robust, delta):
        return f64(L.ba_loss(n(poses), n(points), n(pix), cidx.numpy(), pidx.numpy(), robust, delta))

    def reproj2_accum(nodes, pts, pix, pseg, pa, pb, intr, robust, delta):
        M, u, c = L.reproj2_accum(n(nodes), n(pts), n(pix), pseg.numpy(), pa.numpy(), pb.numpy(), tuple(intr), robust, delta)
        return t(M, nodes), t(u, nodes), f64(c)

    def reproj2_loss(nodes, pts, pix, pseg, pa, pb, intr, robust, delta):
        pe = np.repeat(np.arange(len(pa)), np.diff(pseg.numpy()))
        return f64(L.reproj2_loss(n(nodes), n(pts), n(pix), pa.numpy()[pe], pb.numpy()[pe], tuple(intr), robust, delta))

    torch.library.impl("b200pose::lm_reproj2_accum", "CPU")(reproj2_accum)
    torch.library.impl("b200pose::lm_reproj2_loss", "CPU")(reproj2_loss)

    for name, fn in (("lm_ba_linearize", ba_linearize), ("lm_ba_wtx", ba_wtx), ("lm_ba_wv", ba_wv), ("lm_ba_loss", ba_loss)):
        torch.library.impl(f"b200pose::{name}", "CPU")(fn)

    for name, fn in (("lm_pgo_linearize", pgo_linearize), ("lm_pgo_linearize_w", pgo_linearize_w), ("lm_pgo_scatter", pgo_scatter), ("lm_pgo_spmv", pgo_spmv),
                     ("lm_pgo_loss", pgo_loss)):
        torch.library.impl(f"b200pose::{name}", "CPU")(fn)

    for name, fn in (("lm_poseinv_loss", poseinv_loss), ("lm_poseinv_trial", poseinv_trial),
                     ("lm_reproj_accum", reproj_accum), ("lm_solve6_retract", solve6_retract),
                     ("lm_reproj_loss", reproj_loss), ("lm_reproj_residual", reproj_residual)):
        torch.library.impl(f"b200pose::{name}", "CPU")(fn)


_install_cpu_oracle_lm_kernels()


@pytest.fixture(scope="session")
def golden_lm():
    return np.load(os.path.join(ROOT, "tests", "golden", "lm.npz"))


def _install_cpu_oracle_scan_kernels():
    from pypose_b200.lietensor import scan as _scan  # noqa: F401
    from oracle import scan_oracle as S

    def cumprod(x, group, left):
        return torch.from_numpy(S.cumprod(group, x.detach().double().numpy(), left)).to(x.dtype)

    def imu(dt, gyro, acc, rot, init_rot, gravity):
        n = lambda t: None if t is None else t.detach().double().numpy()
        B, F = dt.shape[:2]
        r = None if rot is None else np.broadcast_to(n(rot), (B, F, 4))
        outs = S.imu_integrate(n(dt), n(gyro), n(acc), r, n(init_rot), gravity)
        return tuple(torch.from_numpy(np.ascontiguousarray(o)).to(dt.dtype) for o in outs)

    def imu_predict(dt, gyro, acc, rot, init_rot, init_pos, init_vel, gravity):
        a, Dp, Dv, Dr, Dt, w = imu(dt, gyro, acc, rot, init_rot, gravity)
        from oracle import lie_oracle as O
        B, F = dt.shape[:2]
        R0 = np.broadcast_to(init_rot.detach().double().numpy().reshape(-1, 1, 4), (B, F, 4))
        p0 = init_pos.detach().double().numpy().reshape(-1, 1, 3)
        v0 = init_vel.detach().double().numpy().reshape(-1, 1, 3)
        rot_o = O.SO3_mul(R0, Dr.double().numpy())
        vel_o = v0 + O.SO3_act(R0, Dv.double().numpy())
        pos_o = p0 + O.SO3_act(R0, Dp.double().numpy()) + v0 * Dt.double().numpy()
        return tuple(torch.from_numpy(np.ascontiguousarray(o)).to(dt.dtype) for o in (rot_o, vel_o, pos_o))

    torch.library.impl("b200pose::cumprod", "CPU")(cumprod)
    torch.library.impl("b200pose::imu_integrate", "CPU")(imu)
    def imu_cov(Rk, Rij, a, dt, gyro_cov, acc_cov, init_cov):
        n = lambda t: t.detach().double().numpy()
        B = dt.shape[0]
        gc = np.broadcast_to(n(gyro_cov), (B,) + tuple(gyro_cov.shape[1:]))
        ac = np.broadcast_to(n(acc_cov), (B,) + tuple(acc_cov.shape[1:]))
        return torch.from_numpy(S.imu_cov(n(Rk), n(Rij), n(a), n(dt), gc, ac, n(init_cov))).to(dt.dtype)

    torch.library.impl("b200pose::imu_predict", "CPU")(imu_predict)
    torch.library.impl("b200pose::imu_full", "CPU")(
        lambda dt, gyro, acc, rot, init_rot, init_pos, init_vel, gravity:
        (*imu(dt, gyro, acc, rot, init_rot, gravity), *imu_predict(dt, gyro, acc, rot, init_rot, init_pos, init_vel, gravity)))
    torch.library.impl("b200pose::imu_cov", "CPU")(imu_cov)


_install_cpu_oracle_scan_kernels()


@pytest.fixture(scope="session")
def golden_scan():
    return np.load(os.path.join(ROOT, "tests", "golden", "scan_imu.npz"))
