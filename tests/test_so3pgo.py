"""CPU checks of the SO3 pose-graph (rotation averaging) route's oracle (oracle/so3pgo_oracle.py): the reference's dense LM
trajectories (tests/golden/so3pgo.npz), the reference's autograd Jacobians, finite differences at small residuals, and a
host build of csrc/so3pgo_math.cuh against the oracle."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import lie_oracle as L
from oracle import so3pgo_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "so3pgo.npz")
CASES = {"constant": ("constant", 0, 1.0), "trustregion": ("trustregion", 0, 1.0), "far": ("trustregion", 0, 1.0),
         "huber": ("trustregion", 1, 0.05), "cauchy": ("trustregion", 3, 0.1), "module": ("trustregion", 0, 1.0)}
_HOST = {}


def golden_case(name):
    g = np.load(GOLDEN)
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_dense_lm_reproduces_reference_trajectory(name):
    g = golden_case(name)
    kind, rk, delta = CASES[name]
    r = S.lm(g["nodes0"], g["Z"], g["edges"], len(g["loss"]), kind, kind=rk, delta=delta)
    np.testing.assert_array_equal(r["reject"], g["reject"])
    np.testing.assert_allclose(r["loss"], g["loss"], rtol=1e-8)
    np.testing.assert_allclose(r["nodes"], g["nodes"], rtol=0, atol=1e-8)


def test_golden_has_a_far_start_and_large_residual_jacobians():
    g = golden_case("far")
    err0 = L.log("SO3", L.mul("SO3", g["nodes0"], L.inv("SO3", g["gt"])))
    assert np.linalg.norm(err0, axis=1).max() > 2.0
    assert np.linalg.norm(golden_case("jac")["r"], axis=1).max() > 3.0


def test_oracle_jacobian_matches_reference_autograd_and_its_fourth_column_is_zero():
    g = golden_case("jac")
    nodes = np.concatenate([g["A"], g["B"]])
    E = len(g["A"])
    edges = np.stack([np.arange(E), E + np.arange(E)], 1)
    J, r = S.jacobian(nodes, g["Z"], edges)
    np.testing.assert_allclose(r, g["r"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(J, g["J"], rtol=0, atol=1e-12 * max(1.0, np.abs(g["J"]).max()))
    np.testing.assert_array_equal(g["J4"][..., 3], 0.0)          # the reference's padded 4th column


def test_oracle_jacobian_matches_finite_differences_at_small_residuals():
    g = golden_case("jac")
    small = np.linalg.norm(g["r"], axis=1) < 0.1
    assert small.sum() >= 8
    A, B, Z = g["A"][small], g["B"][small], g["Z"][small]
    E = len(A)
    nodes, edges = np.concatenate([A, B]), np.stack([np.arange(E), E + np.arange(E)], 1)
    J, _ = S.jacobian(nodes, Z, edges)
    h = 1e-6
    for k in range(3):
        d = np.zeros((E, 3))
        d[:, k] = h
        rp, _ = S.residual(np.concatenate([A, L.mul("SO3", L.exp("SO3", d), B)]), Z, edges)
        rm, _ = S.residual(np.concatenate([A, L.mul("SO3", L.exp("SO3", -d), B)]), Z, edges)
        np.testing.assert_allclose(J[:, :, k], (rp - rm) / (2 * h), rtol=0, atol=1e-7)
        # J_A = -J_B: perturbing the first node
        rp, _ = S.residual(np.concatenate([L.mul("SO3", L.exp("SO3", d), A), B]), Z, edges)
        rm, _ = S.residual(np.concatenate([L.mul("SO3", L.exp("SO3", -d), A), B]), Z, edges)
        np.testing.assert_allclose(-J[:, :, k], (rp - rm) / (2 * h), rtol=0, atol=1e-7)


def test_oracle_node_sums_and_dense_system_agree():
    d = S.problem(9, N=40)
    N = len(d["nodes0"])
    b = S.blocks(d["nodes0"], d["Z"], d["edges"], 3, 0.1)
    Hd, g = S.node_sums(b, d["edges"], N)
    H = S.dense_H(b, d["edges"], N)
    for n in range(N):
        np.testing.assert_allclose(H[3 * n:3 * n + 3, 3 * n:3 * n + 3], Hd[n], rtol=1e-12, atol=1e-12)
    # the 3-unknown step equals the reference's 4-column step
    Hdamp = H.copy()
    k = np.arange(3 * N)
    Hdamp[k, k] = np.clip(Hdamp[k, k], 1e-6, 1e32) * 1.5
    x3 = np.linalg.solve(Hdamp, -g.reshape(-1)).reshape(N, 3)
    D4, _, _ = S.dense_step(d["nodes0"], d["Z"], d["edges"], 1.5, 3, 0.1)
    np.testing.assert_allclose(D4[:, :3], x3, rtol=1e-9, atol=1e-12)
    np.testing.assert_array_equal(D4[:, 3], 0.0)


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="so3pgo_host_")
        so = os.path.join(d, "libso3pgohost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "so3pgo_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data)


def test_host_math_header_matches_oracle():
    """theta = 0, theta <= eps, small and moderate angles and pi - 1e-3 (the reference's Jacobians), plus a graph."""
    g = golden_case("jac")
    d = S.problem(5)
    eye = np.array([[0.0, 0.0, 0.0, 1.0]])                                 # exactly theta = 0
    A = np.ascontiguousarray(np.concatenate([g["A"], d["nodes0"][d["edges"][:, 0]], eye]))
    B = np.ascontiguousarray(np.concatenate([g["B"], d["nodes0"][d["edges"][:, 1]], eye]))
    Z = np.ascontiguousarray(np.concatenate([g["Z"], d["Z"], eye]))
    th = np.linalg.norm(g["r"], axis=1)
    assert (0.0 < th.min() <= np.finfo(float).eps) and th.max() > np.pi - 2e-3
    E = len(A)
    r, J, M, u = np.zeros((E, 3)), np.zeros((E, 3, 3)), np.zeros((E, 6)), np.zeros((E, 3))
    _host().so3pgo_host_edges(_vp(A), _vp(B), _vp(Z), _vp(r), _vp(J), _vp(M), _vp(u), ctypes.c_longlong(E))
    Jo, ro = S.jacobian(np.concatenate([A, B]), Z, np.stack([np.arange(E), E + np.arange(E)], 1))
    np.testing.assert_allclose(r, ro, rtol=0, atol=1e-12)
    np.testing.assert_allclose(J, Jo, rtol=0, atol=1e-11 * np.abs(Jo).max())
    Mo = S.pack(np.swapaxes(Jo, 1, 2) @ Jo)
    np.testing.assert_allclose(M, Mo, rtol=0, atol=1e-11 * np.abs(Mo).max())
    np.testing.assert_allclose(u, np.einsum("eka,ek->ea", Jo, ro), rtol=0, atol=1e-11 * np.abs(Mo).max())


def test_abi_declares_the_so3pgo_entry_points():
    from pypose_b200._optable import lm_symbols
    names = {s for s, _, _ in lm_symbols()}
    for base in ("linearize", "loss", "node_sums", "damp_inv", "pcg", "cg_finish", "predicted"):
        for sfx in ("f32", "f64"):
            assert f"b200_lm_so3pgo_{base}_{sfx}" in names
