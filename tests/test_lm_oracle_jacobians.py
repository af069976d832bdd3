"""The LM oracle's Jacobian blocks against central differences of the oracle's own residuals, in fp64 (no GPU): the
kernels are checked against these blocks (tests/test_lm_linearize_paths_gpu.py), so they must be derivatives of the
residuals and not a restatement of the kernels' formulas.  Also the node-ordered edge layout of the oracle against the one
the library builds (optim/structured.py PGOProblem)."""
import numpy as np
import pytest
import torch

from oracle import lie_oracle as O
from oracle import lm_oracle as L
from tests.util import rand_group

EPS = 1e-6
TOL = 1e-7            # central differences: O(EPS^2) truncation, O(1e-16 / EPS) rounding


def _perturb(X, k, s):
    """Exp(s e_k) X (left perturbation of an SE3 element)."""
    xi = np.zeros((X.shape[0], 6))
    xi[:, k] = s
    return O.mul("SE3", O.exp("SE3", xi), X)


def _fd(res, X, dim=6):
    """(m, d, dim) central differences of res(X') over the left perturbations (SE3, dim 6) or translations (R3, dim 3)."""
    cols = []
    for k in range(dim):
        if dim == 6:
            hi, lo = _perturb(X, k, EPS), _perturb(X, k, -EPS)
        else:
            hi, lo = X.copy(), X.copy()
            hi[:, k] += EPS
            lo[:, k] -= EPS
        cols.append((res(hi) - res(lo)) / (2 * EPS))
    return np.stack(cols, -1)


def test_pgo_jac_blocks_are_derivatives_of_the_residual():
    rng = np.random.default_rng(0)
    E = 200
    A, B = rand_group(rng, "SE3", E, tmax=2.0), rand_group(rng, "SE3", E, tmax=2.0)
    # measurements that leave residual rotations from ~0 up to pi - 0.01
    ang = np.linspace(0.0, np.pi - 0.01, E)
    ax = rng.standard_normal((E, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    R = O.exp("SE3", np.concatenate([0.3 * rng.standard_normal((E, 3)), ax * ang[:, None]], 1))
    Z = O.mul("SE3", O.mul("SE3", O.inv("SE3", A), B), O.inv("SE3", R))
    ei, ej = np.arange(E), np.arange(E, 2 * E)
    nodes = np.concatenate([A, B])
    r, J = L.pgo_jac_blocks(nodes, Z, ei, ej)
    assert np.abs(np.linalg.norm(r[:, 3:], axis=1) - ang).max() < 1e-9
    dB = _fd(lambda X: L.pgo_residual(np.concatenate([A, X]), Z, ei, ej)[0], B)
    dA = _fd(lambda X: L.pgo_residual(np.concatenate([X, B]), Z, ei, ej)[0], A)
    for Jk in (J, L.pgo_jac_blocks(nodes, Z, ei, ej, exact=True)[1]):
        assert np.abs(dB - Jk).max() <= TOL * max(1.0, np.abs(Jk).max())
        assert np.abs(dA + Jk).max() <= TOL * max(1.0, np.abs(Jk).max())


@pytest.mark.parametrize("angle", [0.0, 1e-7, 1e-4, 0.3, 0.999, 1.001, 2.0, np.pi - 0.01])
def test_exact_se3_jl_inv_matches_the_reference_formula(angle):
    """se3_Jl_inv_exact (series below theta = 1) is the reference's Jl^-1: against lie_oracle.se3_Jl_inv evaluated in
    extended precision with its Taylor branch widened to theta < 1e-2, to 1e-14 of the largest entry."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((64, 6))
    x[:, 3:] *= angle / np.linalg.norm(x[:, 3:], axis=1, keepdims=True)
    if np.finfo(np.longdouble).eps > 1e-18:
        pytest.skip("no extended-precision long double on this platform")
    with O.wide_taylor():
        ref = O.se3_Jl_inv(x.astype(np.longdouble)).astype(np.float64)
    assert np.abs(L.se3_Jl_inv_exact(x) - ref).max() <= 1e-14 * np.abs(ref).max()


@pytest.mark.parametrize("intr", [L.README_INTR, (320.0, 0.7, 310.0, 300.0, 250.0)], ids=["readme", "skew"])
def test_reproj2_jac_rows_are_derivatives_of_the_residual(intr):
    rng = np.random.default_rng(1)
    m = 300
    Ta, Tb = rand_group(rng, "SE3", m, tmax=0.5, t_sigma=0.5), rand_group(rng, "SE3", m, tmax=0.5, t_sigma=0.5)
    y = rng.uniform([-2, -2, 2], [2, 2, 6], (m, 3))
    pts = O.act("SE3", O.mul("SE3", O.inv("SE3", Ta), Tb), y)        # T_b^-1 T_a p = y: in front of camera b
    pix = rng.standard_normal((m, 2))
    ia, ib = np.arange(m), np.arange(m, 2 * m)
    nodes = np.concatenate([Ta, Tb])
    J = L.reproj2_jac_rows(nodes, pts, ia, ib, intr)
    da = _fd(lambda X: L.reproj2_residual(np.concatenate([X, Tb]), pts, pix, ia, ib, intr)[0], Ta)
    db = _fd(lambda X: L.reproj2_residual(np.concatenate([Ta, X]), pts, pix, ia, ib, intr)[0], Tb)
    scale = max(1.0, np.abs(J).max())
    assert np.abs(da - J).max() <= TOL * scale
    assert np.abs(db + J).max() <= TOL * scale


def test_ba_jac_rows_are_derivatives_of_the_residual():
    rng = np.random.default_rng(2)
    m = 300
    T = rand_group(rng, "SE3", m, tmax=0.5, t_sigma=0.5)
    y = rng.uniform([-2, -2, 2], [2, 2, 6], (m, 3))
    p = O.act("SE3", O.inv("SE3", T), y)
    pix = rng.standard_normal((m, 2))
    idx = np.arange(m)
    Jc, Jp = L.ba_jac_rows(T, p, idx, idx)
    dc = _fd(lambda X: L.ba_residual(X, p, pix, idx, idx), T)
    dp = _fd(lambda X: L.ba_residual(T, X, pix, idx, idx), p, dim=3)
    assert np.abs(dc - Jc).max() <= TOL * max(1.0, np.abs(Jc).max())
    assert np.abs(dp - Jp).max() <= TOL * max(1.0, np.abs(Jp).max())
    # the rows rebuilt from y = T p and sqrt(rho') (the Y4 layout of the deterministic BA kernels) are the same rows
    sw = rng.uniform(0.2, 1.0, m)
    Jc_y, Jp_y = L.ba_rows_from_y(O.act("SE3", T, p), sw, T, idx)
    assert np.abs(Jc_y - Jc * sw[:, None, None]).max() <= 1e-12 * np.abs(Jc).max()
    assert np.abs(Jp_y - Jp * sw[:, None, None]).max() <= 1e-12 * np.abs(Jp).max()


def test_predicted_oracles_match_the_dense_quadratic_model():
    rng = np.random.default_rng(3)
    N, E = 30, 80
    ei, ej = rng.integers(0, N, E), rng.integers(0, N, E)
    B = rng.standard_normal((E, 6, 6))
    M21 = L._triu_pack(B @ np.swapaxes(B, -1, -2))
    u, x = rng.standard_normal((E, 6)), rng.standard_normal((N, 6))
    H = np.zeros((6 * N, 6 * N))
    Mb = L._triu_unpack(M21)
    for e in range(E):
        for a, sa in ((ei[e], 1), (ej[e], -1)):
            for b, sb in ((ei[e], 1), (ej[e], -1)):
                H[6 * a:6 * a + 6, 6 * b:6 * b + 6] += sa * sb * Mb[e]
    Hd, g = L.pgo_scatter(M21, u, ei, ej, N)
    xv = x.reshape(-1)
    val, terms = L.pgo_predicted(M21, u, ei, ej, x, terms=True)
    np.testing.assert_allclose(val, xv @ H @ xv + 2 * xv @ g.reshape(-1), rtol=1e-12)
    assert terms >= abs(val)
    C, P, m = 5, 12, 40
    Jc, Jp, rs = rng.standard_normal((m, 12)), rng.standard_normal((m, 6)), rng.standard_normal((m, 2))
    cidx, pidx = rng.integers(0, C, m), rng.integers(0, P, m)
    xc, xp = rng.standard_normal((C, 6)), rng.standard_normal((P, 3))
    from tests.test_lm_gpu import _ba_sparse_J
    Jsp = _ba_sparse_J(Jc, Jp, cidx, pidx, C, P)
    d = np.concatenate([xc.reshape(-1), xp.reshape(-1)])
    Jd = Jsp @ d
    val, terms = L.ba_predicted(Jc, Jp, rs, cidx, pidx, xc, xp, terms=True)
    np.testing.assert_allclose(val, Jd @ (2 * rs.reshape(-1) + Jd), rtol=1e-12)
    assert terms >= abs(val)


def test_node_layout_matches_the_library():
    from pypose_b200.lietensor import SE3
    from pypose_b200.optim.structured import PGOProblem
    rng = np.random.default_rng(4)
    N, E = 50, 300
    ei, ej = rng.integers(0, N, E), rng.integers(0, N, E)
    ei[:5], ej[:5] = 3, 7                              # a repeated edge
    ei[5:8], ej[5:8] = 9, 2                            # ei > ej
    keep = ei != ej
    ei, ej = ei[keep], ej[keep]
    ei[ei == 49], ej[ej == 49] = 0, 1                  # node 49 isolated
    edges = torch.from_numpy(np.stack([ei, ej], 1))
    prob = PGOProblem(None, edges, None, None, None, (0, 1.0), 1e-6, 10,
                      param=SE3(torch.from_numpy(rand_group(rng, "SE3", N))))
    epos_i, epos_j, nptr, nother = L.node_layout(ei, ej, N)
    for mine, lib in ((epos_i, prob.epos_i), (epos_j, prob.epos_j), (nptr, prob.nptr), (nother, prob.nother)):
        assert np.array_equal(mine, lib.numpy())
    assert nptr[49] == nptr[50]
    # every slot is owned by exactly one (edge, end), inside its node's range
    assert np.array_equal(np.sort(np.concatenate([epos_i, epos_j])), np.arange(2 * len(ei)))
    assert ((nptr[ei] <= epos_i) & (epos_i < nptr[ei + 1])).all() and ((nptr[ej] <= epos_j) & (epos_j < nptr[ej + 1])).all()
    assert np.array_equal(nother[epos_i], ej) and np.array_equal(nother[epos_j], ei)
