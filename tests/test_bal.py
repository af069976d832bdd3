"""BAL bundle adjustment without a GPU: the fp64 oracle (oracle/bal_oracle.py) against the reference's dense LM
trajectories (tests/golden/bal.npz, oracle/make_golden_bal.py), its analytic Jacobian rows against finite differences,
and a host build of csrc/bal_math.cuh against the oracle."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import bal_oracle as B
from oracle import lie_oracle as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "bal.npz")
CASES = {"constant": "constant", "trustregion": "trustregion", "reject": "trustregion"}
_HOST = {}


def golden_case(name):
    g = np.load(GOLDEN)
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_dense_lm_reproduces_reference_trajectory(name):
    g = golden_case(name)
    r = B.lm(g["K0"], g["T0"], g["P0"], g["pix"], g["cidx"], g["pidx"], len(g["loss"]), CASES[name])
    np.testing.assert_array_equal(r["reject"], g["reject"])
    np.testing.assert_allclose(r["loss"], g["loss"], rtol=1e-8)      # the far start amplifies rounding
    np.testing.assert_allclose(r["K"], g["K"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(r["T"], g["T"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(r["P"], g["P"], rtol=0, atol=1e-8)


def test_golden_has_a_rejected_trial():
    assert golden_case("reject")["reject"].sum() > 0


def test_oracle_rows_match_finite_differences():
    d = B.problem(3)
    K, T, P, pix, ci, pi_ = d["K0"], d["T0"], d["P0"], d["pix"], d["cidx"], d["pidx"]
    Jc, Jp = B.rows(K, T, P, ci, pi_)
    h = 1e-6
    for a in range(9):                         # camera columns: left SE3 perturbation, then f, k1, k2
        e = np.zeros(9)
        e[a] = h
        cols = []
        for s in (1, -1):
            xc = np.tile(s * e, (len(K), 1))
            Kt, Tt, _ = B.retract(K, T, P, xc, np.zeros_like(P))
            cols.append(B.residual(Kt, Tt, P, pix, ci, pi_))
        fd = (cols[0] - cols[1]) / (2 * h)
        np.testing.assert_allclose(Jc[:, :, a], fd, rtol=1e-5, atol=1e-5 * np.abs(fd).max())
    for a in range(3):
        e = np.zeros(3)
        e[a] = h
        fd = (B.residual(K, T, P + e, pix, ci, pi_) - B.residual(K, T, P - e, pix, ci, pi_)) / (2 * h)
        np.testing.assert_allclose(Jp[:, :, a], fd, rtol=1e-5, atol=1e-5 * np.abs(fd).max())


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="bal_host_")
        so = os.path.join(d, "libbalhost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "bal_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data)


def test_host_rows_blocks_and_inverse_match_oracle():
    d = B.problem(4)
    K, T, P, ci, pi_ = d["K0"], d["T0"], d["P0"], d["cidx"], d["pidx"]
    y = np.ascontiguousarray(L.act("SE3", T[ci], P[pi_]))
    q, Kc = np.ascontiguousarray(T[ci, 3:]), np.ascontiguousarray(K[ci])
    m = len(ci)
    jc, jp = np.zeros((m, 2, 9)), np.zeros((m, 2, 3))
    _host().bal_host_rows(_vp(y), _vp(q), _vp(Kc), ctypes.c_double(0.75), _vp(jc), _vp(jp), ctypes.c_longlong(m))
    Jc, Jp = B.rows(K, T, P, ci, pi_)
    np.testing.assert_allclose(jc, 0.75 * Jc, rtol=1e-10, atol=1e-10 * np.abs(Jc).max())
    np.testing.assert_allclose(jp, 0.75 * Jp, rtol=1e-10, atol=1e-10 * np.abs(Jp).max())
    # one camera's 45-word block, a packed mat-vec and the damped inverse
    rows = np.ascontiguousarray(Jc[ci == 0])
    H45 = np.zeros(45)
    _host().bal_host_sum_rows(_vp(rows), _vp(H45), ctypes.c_longlong(len(rows)))
    H = np.einsum("kia,kib->ab", rows, rows)
    iu = np.triu_indices(9)
    np.testing.assert_allclose(H45, H[iu], rtol=1e-12, atol=1e-12 * np.abs(H).max())
    x = np.random.default_rng(0).normal(size=9)
    yv, Hinv = np.zeros(9), np.zeros(45)
    _host().bal_host_block(_vp(H45), _vp(x), ctypes.c_double(1.5), ctypes.c_double(1e-6), ctypes.c_double(1e32), _vp(yv),
                           _vp(Hinv))
    np.testing.assert_allclose(yv, H @ x, rtol=1e-12, atol=1e-12 * np.abs(H @ x).max())
    inv = np.linalg.inv(B.damp(H, 1.5, 1e-6, 1e32))
    np.testing.assert_allclose(Hinv, inv[iu], rtol=1e-8, atol=1e-10 * np.abs(inv).max())


def test_abi_declares_the_bal_entry_points():
    from pypose_b200._optable import lm_symbols
    text = open(os.path.join(ROOT, "include", "b200pose.h")).read()
    declared = set(re.findall(r"^int\s+(b200_lm_bal_\w+)\s*\(", text, flags=re.M))
    bases = ["linearize_seg", "point_blocks", "wv_seg", "schur_diag_seg", "wtx_gather", "damp_inv", "pcg", "cg_finish",
             "predicted", "loss", "retract"]
    want = {f"b200_lm_bal_{b}_{s}" for b in bases for s in ("f32", "f64")}
    assert declared == want
    assert want <= {s for s, *_ in lm_symbols()}
