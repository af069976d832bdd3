"""The width-generic PCGs on every launch path, in fp32 and fp64:

  * the node-ordered two-kernel iteration of csrc/pcg2.cu at W = 3 (SO3), 6 (SE3) and 7 (Sim3 nodes): node sums, solve
    against fp64 sparse solves, chunk invariance, every stop reason of the best-iterate guard and the edge inputs, in
    each grid regime of lm_grid (below);
  * the BAL reduced-camera PCG of csrc/bal.cu at W = 9 on both edges of its two single-CTA kernels and the grid path;
  * the one-call LM trial of csrc/lmdrive.cu (b200_lm_pgo2_step, families 0, 2 and 3) against the Python-driven trial,
    bit for bit, including rejected trials and a maxiter that is not a multiple of the chunk size.

Grid regimes of the node-ordered iteration.  lm_grid runs 128 threads per CTA and caps a grid at 8 CTAs per SM; the node
sums and operator kernels give 4 lanes to a node (32 nodes per CTA and pass), cg_update one thread to a node (128 per CTA
and pass):
  (a) one CTA for both kernels;
  (b) several CTAs, one pass of every grid-stride loop;
  (c) cg_update on more than 384 CTAs (reduce_sums folds the CTA partials 4 at a time), operator and node sums multi-pass;
  (d) cg_update multi-pass.
N is derived from the device's SM count and every test asserts the regime it reached."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch

import pypose_b200 as pp
from oracle import bal_oracle as B
from oracle import lie_oracle as O
from pypose_b200.optim import _fused, _lmstep, structured
from pypose_b200.optim.solver import PCG
from tests.test_bal_gpu import Layout
from tests.test_lm_gpu import (CG_DONE, CG_ITERS, CG_PATIENCE, CG_RR, PCG_DT, UNIT_ROUNDOFF, _check_pcg, _damped,
                               _dense_sym)

pytestmark = pytest.mark.gpu
STOP_SCALES = (1.0 + 1e-3, 1.0 + 1e-5, 1.0 + 1e-7, 1.0 + 1e-9)     # damping of the stop-reason systems, most damped first
THREADS, CTAS_PER_SM, LANES = 128, 8, 4        # csrc/lm_common.cuh lm_grid, csrc/pcg2.cu kLanes
# block width W -> (group, problem kind, parameter width D, LieTensor constructor)
GROUPS = {3: ("SO3", "so3", 4, pp.SO3), 6: ("SE3", "pgo", 7, pp.SE3), 7: ("Sim3", "sim3", 8, pp.Sim3)}


def cu(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


def _cdiv(a, b):
    return -(-a // b)


def _cap():
    return CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count


def _node_regime(N):
    """Launch geometry of the node-ordered iteration at N nodes: (operator CTAs, passes), (cg_update CTAs, passes)."""
    cap = _cap()
    op, vec = min(_cdiv(N, THREADS // LANES), cap), min(_cdiv(N, THREADS), cap)
    return op, _cdiv(_cdiv(N, THREADS // LANES), op), vec, _cdiv(_cdiv(N, THREADS), vec)


def _regime_size(regime):
    """An odd N, not a multiple of 32, that reaches the regime on this device."""
    cap = _cap()
    N = {"a": 29, "b": 3001, "c": max(2 * 32 * cap, 385 * THREADS) + 1, "d": int(1.05 * cap * THREADS) | 1}[regime]
    op, op_pass, vec, vec_pass = _node_regime(N)
    reached = {"a": op == vec == 1,
               "b": op > 1 and vec > 1 and op_pass == vec_pass == 1,
               "c": vec > 384 and vec_pass == 1 and op_pass > 1,
               "d": vec_pass > 1}[regime]
    assert N % 2 == 1 and reached, (regime, N, op, op_pass, vec, vec_pass)
    return N, f"N={N} operator {op} CTAs x {op_pass} passes, cg_update {vec} CTAs x {vec_pass} passes"


def _graph(W, N, rng, loops=None, span=20, noise=0.1, meas=0.02, at_measurements=False):
    """A chain plus `loops` banded loop closures (nodes at most `span` apart) on random absolute nodes of the group of
    width W (Sim3 scales within e^+-0.4); the start is the ground truth perturbed by Exp(noise).  at_measurements: every
    node and measurement is the identity, so every residual is exactly 0.  Returns nodes (N,D), edges (E,2), Z (E,D)."""
    grp, _, D, _ = GROUPS[W]
    loops = N // 2 if loops is None else loops
    span = min(span, N - 1)
    ci = rng.integers(0, N - span, loops) if span >= 2 else np.zeros(0, np.int64)
    cj = ci + rng.integers(2, span + 1, len(ci)) if span >= 2 else ci
    edges = np.stack([np.concatenate([np.arange(N - 1), ci]), np.concatenate([np.arange(1, N), cj])], 1).astype(np.int64)
    if at_measurements:
        eye = O.exp(grp, np.zeros((1, W)))
        return np.repeat(eye, N, 0), edges, np.repeat(eye, len(edges), 0)
    tangent = rng.normal(0, 1.0, (N, W))
    if W == 7:
        tangent[:, 6] *= 0.2
    gt = O.exp(grp, tangent)
    Z = O.mul(grp, O.mul(grp, O.inv(grp, gt[edges[:, 0]]), gt[edges[:, 1]]), O.exp(grp, meas * rng.normal(size=(len(edges), W))))
    return O.mul(grp, O.exp(grp, noise * rng.normal(size=(N, W))), gt), edges, Z


def _problem(W, nodes, edges, Z, dt):
    """The structured problem of the width-W family (its node adjacency: nptr, nother, epos_i / epos_j)."""
    _, kind, _, lt = GROUPS[W]
    model = pp.module.PoseGraph(lt(cu(nodes, dt)))
    e, Zt = torch.from_numpy(edges).cuda(), lt(cu(Z, dt))
    if W == 6:
        return structured.PGOProblem(model, e, Zt, None, None, (0, 1.0), 1e-12, None)
    cls = structured.SO3PGOProblem if W == 3 else structured.Sim3PGOProblem
    return cls(model, e, Zt, None, (0, 1.0), 1e-12, None)


def _linearize(prob, W):
    """_fused.pgo_linearize_nodes with the per-slot gradients `un` kept: Mn, un, Hd, g."""
    spec, nodes = _fused.NODE_WIDTHS[W], prob._nodes()
    E, N, dt = prob.ei.shape[0], prob.nptr.shape[0] - 1, nodes.dtype
    Mn = torch.empty(2 * E, spec.slot, dtype=dt, device="cuda")
    un = torch.empty(2 * E, W, dtype=dt, device="cuda")
    p = _fused._p
    _fused._launch(_fused._EDGE_LINEARIZE[prob.kind], nodes, [p(nodes), p(prob.Z), p(prob.ei), p(prob.ej), p(prob.epos_i),
                                                              p(prob.epos_j), p(Mn), p(un), p(_fused._workspace(nodes.device)),
                                                              0, 1.0], E)
    Hd = torch.empty(N, spec.packed, dtype=dt, device="cuda")
    g = torch.empty(N, W, dtype=dt, device="cuda")
    _fused._launch(spec.node_sums, nodes, [p(Mn), p(un), p(prob.nptr), p(Hd), p(g)], N)
    return Mn, un, Hd, g


def _sparse_H(Hd, Mn, nptr, nother, W):
    """fp64 block-sparse H from the node-ordered blocks: row n holds the diagonal block Hd[n] and -Mn[s] at column block
    nother[s] for each of its slots s."""
    N, S, PW = len(Hd), len(Mn), W * (W + 1) // 2
    deg = np.diff(nptr)
    indptr = nptr.astype(np.int64) + np.arange(N + 1)
    slot_pos = np.arange(S) + np.repeat(np.arange(N), deg) + 1
    data, indices = np.empty((N + S, W, W)), np.empty(N + S, np.int64)
    data[indptr[:-1]], indices[indptr[:-1]] = _dense_sym(Hd, N, W), np.arange(N)
    data[slot_pos], indices[slot_pos] = -_dense_sym(Mn[:, :PW], S, W), nother
    return sp.bsr_matrix((data, indices, indptr), shape=(W * N, W * N))


def _np(t):
    return t.double().cpu().numpy()


class NodeSystem:
    """(H + clamp/damping) x = -g on node-ordered blocks through the width-W entry points, as _fused.pgo_solve_nodes
    enqueues them, with the chunking chosen by the caller.  Mn_op: the blocks of the operator (the preconditioner always
    comes from Hd)."""

    def __init__(self, W, Mn, nother, nptr, Hd, g, scale, dmin=1e-6, dmax=1e32, Mn_op=None):
        self.spec, self.W, self.n = _fused.NODE_WIDTHS[W], W, Hd.shape[0]
        self.Mn, self.Mn_op, self.nother, self.nptr, self.b = Mn, Mn if Mn_op is None else Mn_op, nother, nptr, g
        dt = Hd.dtype
        self.extra, self.Minv, self.Hdamp = torch.empty_like(g), torch.empty_like(Hd), torch.empty_like(Hd)
        p = _fused._p
        _fused._launch(self.spec.damp_inv, Hd, [p(Hd), float(scale), float(dmin), float(dmax), p(self.Hdamp), p(self.extra),
                                                p(self.Minv)], self.n)
        self.x, self.r, self.z, self.p0, self.p1, self.q, self.xbest = (torch.zeros_like(g) for _ in range(7))
        self.cg = torch.zeros(16, dtype=torch.float64, device="cuda")
        self.dt = dt

    def pcg(self, first, iters, tol, maxiter):
        p = _fused._p
        _fused._launch(self.spec.pcg, self.Mn, [p(self.Mn_op), p(self.nother), p(self.nptr), p(self.Minv), p(self.extra),
                                                p(self.b), p(self.x), p(self.r), p(self.z), p(self.p0), p(self.p1), p(self.q),
                                                p(self.xbest), p(self.cg), p(_fused._workspace(self.Mn.device)), float(tol),
                                                int(maxiter), int(first), int(iters)], self.n)

    def finish(self):
        p = _fused._p
        _fused._launch(self.spec.cg_finish, self.Mn, [p(self.x), p(self.xbest), p(self.cg)], self.n)

    def predicted(self, x):
        """operator mode 1: x^T H x + 2 x^T g (fp64 on the device)."""
        p, ws = _fused._p, _fused._workspace(self.Mn.device)
        _fused._launch(self.spec.predicted, self.Mn, [p(self.Mn), p(self.nother), p(self.nptr), p(x), p(self.b), p(ws)], self.n)
        return ws[:1].clone()


class BalSystem:
    """The damped reduced camera system of _fused.bal_solve (S = Hc - W Hpp^-1 W^T, rhs from gc and gp) through
    b200_lm_bal_pcg / b200_lm_bal_cg_finish, with the chunking chosen by the caller.  negate: -Hc is passed as the
    block-diagonal part of the operator."""

    def __init__(self, lay, K, T, Y4s, Hcc, Hpp, gc, gp, scale, dmin=1e-6, dmax=1e32, negate=False):
        p = _fused._p
        self.Y4, self.Y4p = Y4s
        cseg, split, tpi, _, self.cidx_p, self.pptr, _ = lay.geom
        C, P, dt = Hcc.shape[0], Hpp.shape[0], Hcc.dtype
        self.n, self.P, self.m, self.dt = C, P, self.Y4.shape[0], dt
        self.seg = [p(self.Y4), p(T), p(K), p(lay.pidx), p(cseg), split, tpi]
        self.Hc, self.Minv = torch.empty(C, 45, dtype=dt, device="cuda"), torch.empty(C, 45, dtype=dt, device="cuda")
        self.Hpinv = torch.empty(P, 6, dtype=dt, device="cuda")
        self.part = torch.empty(C * split, 45, dtype=dt, device="cuda") if split > 1 else None
        _fused._launch("b200_lm_bal_damp_inv", self.Y4, [p(Hcc), float(scale), float(dmin), float(dmax), p(self.Hc), None], C)
        _fused._launch("b200_lm_pt3_damp_inv", self.Y4, [p(Hpp), float(scale), float(dmin), float(dmax), p(self.Hpinv)], P)
        Sd = self.Hc.clone()
        _fused._launch("b200_lm_bal_schur_diag_seg", self.Y4, [*self.seg, p(self.Hpinv), p(Sd), p(self.part)], C)
        self.b = gc.clone()
        _fused._launch("b200_lm_bal_wv_seg", self.Y4, [*self.seg, p(self.Hpinv), p(gp), p(self.b), p(self.part)], C)
        _fused._launch("b200_lm_bal_damp_inv", self.Y4, [p(Sd), 1.0, -3.0e38, 3.0e38, None, p(self.Minv)], C)
        self.D = -self.Hc if negate else self.Hc
        self.x, self.r, self.z, self.p, self.q, self.xbest = (torch.zeros(C, 9, dtype=dt, device="cuda") for _ in range(6))
        self.t = torch.empty(P, 3, dtype=dt, device="cuda")
        self.cg = torch.zeros(16, dtype=torch.float64, device="cuda")

    def pcg(self, first, iters, tol, maxiter):
        p = _fused._p
        _fused._launch("b200_lm_bal_pcg", self.Y4, [
            *self.seg, self.m, p(self.Y4p), p(self.cidx_p), p(self.pptr), p(self.D), p(self.Hpinv), p(self.Minv), p(self.b),
            p(self.x), p(self.r), p(self.z), p(self.p), p(self.q), p(self.t), p(self.part), p(self.xbest), p(self.cg),
            p(_fused._workspace(self.Y4.device)), float(tol), int(maxiter), self.P, int(first), int(iters)], self.n)

    def finish(self):
        p = _fused._p
        _fused._launch("b200_lm_bal_cg_finish", self.Y4, [p(self.x), p(self.xbest), p(self.cg)], self.n)


def _solve(sys_, tol, maxiter, chunks, patience=None):
    """Enqueue the PCG in chunks (first chunk sizes, the last one repeated) until the device reports done or maxiter
    iterations are enqueued, as _fused._run_chunks does, then cg_finish.  With chunks [1] every iterate x_0 = 0, x_1, ...
    and |r_k|^2 are recorded.  `patience`, if given, replaces the stagnation patience after the first call.
    Returns x before and after cg_finish, the 16-double state, the iterates and |r_k|^2."""
    record = list(chunks) == [1]
    xs, rr = [sys_.x.clone()], [float((sys_.b.double() ** 2).sum())]
    it, calls = 0, 0
    while True:
        k = max(1, min(chunks[min(calls, len(chunks) - 1)], maxiter - it))
        sys_.pcg(it, k, tol, maxiter)
        it, calls = it + k, calls + 1
        st = sys_.cg.tolist()
        if record and st[CG_ITERS] == it:
            xs.append(sys_.x.clone())
            rr.append(st[CG_RR])
        if calls == 1 and patience is not None:
            sys_.cg[CG_PATIENCE] = patience
        if st[CG_DONE] != 0.0 or it >= maxiter:
            break
    last = sys_.x.clone()
    sys_.finish()
    return last, sys_.x.clone(), sys_.cg.clone(), xs, np.array(rr)


def _chunk_invariance(make, tol, maxiter, tag):
    """The final x, cg_finish's output and the state are bit-identical for one call, chunks of 1, 3 and 8 and a first chunk
    larger than the iterations needed: the kernel sequence does not depend on the chunking.  Returns the one-call run."""
    ref = _solve(make(), tol, maxiter, [maxiter])
    iters = int(ref[2][CG_ITERS].item())
    assert 0 < iters <= maxiter and ref[2][CG_DONE].item() != 0.0, (tag, ref[2].tolist())
    for chunks in ([1], [3], [8], [iters + 7, 8]):
        got = _solve(make(), tol, maxiter, chunks)
        for a, b, what in zip(got[:3], ref[:3], ("x", "cg_finish x", "state")):
            assert torch.equal(a, b), (tag, chunks, what)
    return ref


def _stop_reasons(make, make_negated, quad, tag, conv_tol=1e-4):
    """test_lm_gpu.py test_pcg_guard_stop_reasons_return_the_best_iterate on another system: converged (1), maxiter (4)
    after 3 iterations / after |r| rose / after it fell, stagnated (3) and breakdown (2), each returning its documented
    iterate bit for bit.  make(scale): the system damped by `scale`; quad(scale, x): its quadratic model
    x^T A x + 2 x^T b (None: not checked).  The maxiter and stagnation cases need a |r| that is not monotone: the most
    damped system of STOP_SCALES on which, within 1000 iterations, |r| rises and then reaches a new minimum, and two
    iterations in a row bring no new minimum, is used."""
    run = lambda scale, tol, maxiter, **kw: _solve(make(scale), tol, maxiter, [1], **kw)[1:]
    x, st, xs, rr = run(STOP_SCALES[0], conv_tol, 20_000)
    assert st[CG_DONE] == 1.0 and st[CG_ITERS] == len(xs) - 1 and torch.equal(x, xs[-1]), tag
    for scale in STOP_SCALES:
        x, st, xs, rr = run(scale, 1e-30, 1000)
        prior = np.minimum.accumulate(rr)
        rose = next((k for k in range(2, len(rr)) if rr[k] > 1.01 * prior[k - 1]), None)
        fell = next((k for k in range(rose + 1, len(rr)) if rr[k] < 0.99 * prior[k - 1]), None) if rose else None
        stalled = next((k for k in range(2, len(rr)) if rr[k - 1] >= prior[k - 2] and rr[k] >= prior[k - 2]), None)
        if fell is not None and stalled is not None:
            break
    assert fell is not None and stalled is not None, (tag, "|r| not monotone enough in 1000 iterations", rr)
    run = lambda tol, maxiter, _run=run, **kw: _run(scale, tol, maxiter, **kw)
    for K in (3, rose, fell):
        x, st, xs, rr = run(1e-30, K)
        best = int(np.argmin(rr))
        assert st[CG_DONE] == 4.0 and st[CG_ITERS] == K and len(rr) == K + 1, (tag, K, st.tolist())
        if K != 3:
            assert (best < K) == (K == rose), (tag, K, best, rr)
        assert torch.equal(x, xs[best]), (tag, K, best)
        if quad is not None:
            assert quad(scale, _np(x).reshape(-1)) < 0, (tag, K)
    x, st, xs, rr = run(1e-30, 3000, patience=2.0)
    stop, since = None, 0
    for k in range(1, len(rr)):
        since = 0 if rr[k] < rr[:k].min() else since + 1
        if since >= 2:
            stop = k
            break
    assert stop == stalled and st[CG_DONE] == 3.0 and st[CG_ITERS] == stop == len(rr) - 1, (tag, stop, st.tolist())
    assert torch.equal(x, xs[int(np.argmin(rr))]), tag
    # breakdown: an indefinite operator with an SPD preconditioner stops in the first iteration with x = 0
    x, st, xs, rr = _solve(make_negated(scale), 1e-4, 100, [1])[1:]
    assert st[CG_DONE] == 2.0 and st[CG_ITERS] == 0.0 and len(xs) == 1, (tag, st.tolist())
    assert torch.equal(x, torch.zeros_like(x)), tag
    print(f"{tag}: scale 1 + {scale - 1:.0e}: |r| rose at {rose}, fell at {fell}, stagnated at {stop}")


# ------------------------------------------------------------------------------------------- A. node-ordered PCG, W = 3, 6, 7
@pytest.mark.parametrize("regime", ["a", "b", "c", "d"])
@pytest.mark.parametrize("W", [3, 6, 7])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_node_pcg_in_every_grid_regime(dtn, W, regime):
    """Node sums against an fp64 segment sum of the kernel's own slots; the solve against the bounds of
    test_lm_gpu._check_pcg (and an fp64 sparse LU where that is cheap); the predicted reduction against fp64; chunk
    invariance of x, cg_finish's output and the state; all of it bit-identical to _fused.pgo_solve_nodes."""
    dt, scale, tol = PCG_DT[dtn]
    dmin, dmax, maxiter = 1e-6, 1e32, 20_000
    N, where = _regime_size(regime)
    tag = f"W={W} {dtn} regime ({regime}) {where}"
    nodes, edges, Z = _graph(W, N, np.random.default_rng(40 + W))
    prob = _problem(W, nodes, edges, Z, dt)
    Mn, un, Hd, g = _linearize(prob, W)
    Mn2, Hd2, g2, _ = _fused.pgo_linearize_nodes(prob.kind, prob, prob._nodes(), 0, 1.0)
    PW = W * (W + 1) // 2                   # the SE3 linearisation leaves the 3 padding words of a 24-word slot unwritten
    assert torch.equal(Mn[:, :PW], Mn2[:, :PW]) and torch.equal(Hd, Hd2) and torch.equal(g, g2), tag     # no atomics
    # node sums: each node's sum of its slots, in any order, is within deg * u * (sum of |terms|) of the fp64 sum
    nptr, nother = prob.nptr.cpu().numpy(), prob.nother.cpu().numpy()
    deg, u = np.diff(nptr), UNIT_ROUNDOFF[dt]
    assert deg.min() >= 1
    for got, terms in ((Hd, Mn[:, :PW]), (g, un)):
        t = _np(terms)
        ref, mag = np.add.reduceat(t, nptr[:-1]), np.add.reduceat(np.abs(t), nptr[:-1])
        err = np.abs(_np(got) - ref)
        assert (err <= 2 * u * deg[:, None] * mag).all(), (tag, err.max())
    # the solve
    Hn = _np(Hd)
    H = _sparse_H(Hn, _np(Mn), nptr, nother, W)
    A = _damped(H, scale, dmin, dmax)
    gv = _np(g).reshape(-1)
    make = lambda: NodeSystem(W, Mn, prob.nother, prob.nptr, Hd, g, scale, dmin, dmax)
    _, x, st, _, _ = _chunk_invariance(make, tol, maxiter, tag)
    assert st[CG_DONE].item() == 1.0, (tag, st.tolist())
    xl, iters, pred = _fused.pgo_solve_nodes(Mn, prob.nother, prob.nptr, Hd, g, scale, dmin, dmax, tol, maxiter)
    assert torch.equal(xl, x) and iters == int(st[CG_ITERS].item()), tag
    xv = _np(x).reshape(-1)
    xref = spla.spsolve(A.tocsc(), -gv) if N <= 5000 else None
    _check_pcg(f"{tag} iters={iters}", H, A, gv, xv, xref, scale, tol, dt, 1e-8)
    # predicted reduction (operator mode 1) at the solution
    assert torch.equal(pred, make().predicted(x)), tag
    want = xv @ (H @ xv) + 2 * xv @ gv
    if dt == torch.float64:
        np.testing.assert_allclose(pred.item(), want, rtol=1e-9)
    else:
        assert abs(pred.item() - want) <= 5e-4 * (1 + abs(want) + abs(xv @ (abs(H) @ abs(xv)))), (tag, pred.item(), want)
    print(tag, f"iters={iters}")


@pytest.mark.parametrize("N", [91, 5001])                  # the sizes of test_lm_gpu's W = 6 stop-reason test
@pytest.mark.parametrize("W", [3, 6, 7])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_node_pcg_stop_reasons_return_the_best_iterate(dtn, W, N):
    """Every stop reason of the guard through the node-ordered iteration (p = z + beta p and p.Ap folded into the operator
    kernel, parity of the r.z slots from the iteration index), one iteration per call."""
    dt = PCG_DT[dtn][0]
    op, op_pass, vec, vec_pass = _node_regime(N)
    tag = f"W={W} {dtn} N={N} operator {op} CTAs x {op_pass}, cg_update {vec} CTAs x {vec_pass}"
    nodes, edges, Z = _graph(W, N, np.random.default_rng(50 + W), loops=min(N, 300), span=30)
    prob = _problem(W, nodes, edges, Z, dt)
    Mn, _, Hd, g = _linearize(prob, W)
    make = lambda scale, Mn_op=None: NodeSystem(W, Mn, prob.nother, prob.nptr, Hd, g, scale, Mn_op=Mn_op)
    H = _sparse_H(_np(Hd), _np(Mn), prob.nptr.cpu().numpy(), prob.nother.cpu().numpy(), W)
    gv = _np(g).reshape(-1)
    quad = lambda scale, xv: xv @ (_damped(H, scale, 1e-6, 1e32) @ xv) + 2 * xv @ gv
    # breakdown: with the slots negated the operator is -H + extra, which is indefinite
    _stop_reasons(make, lambda scale: make(scale, -Mn), quad, tag)


@pytest.mark.parametrize("W", [3, 6, 7])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_node_pcg_edge_inputs(dtn, W):
    """g exactly 0 (every node at its measurements): done at init with x = 0 and 0 iterations.  An isolated node: its
    block clamps to dmin * scale and its rows of x stay 0.  A single edge (N = 2).  The state stays finite throughout."""
    dt, scale, tol = PCG_DT[dtn]
    dmin, dmax, maxiter = 1e-6, 1e32, 2000
    rng = np.random.default_rng(60 + W)
    # g = 0
    prob = _problem(W, *_graph(W, 29, rng, at_measurements=True), dt)
    Mn, _, Hd, g = _linearize(prob, W)
    assert torch.count_nonzero(g) == 0 and Hd.abs().max() > 0
    s = NodeSystem(W, Mn, prob.nother, prob.nptr, Hd, g, scale, dmin, dmax)
    _, x, st, _, _ = _solve(s, tol, maxiter, [8])
    assert st[CG_DONE] == 1.0 and st[CG_ITERS] == 0.0 and torch.isfinite(st).all(), st.tolist()
    assert torch.count_nonzero(x) == 0 and s.predicted(x).item() == 0.0
    # an isolated node (the last) next to a connected graph, and a single edge
    for name, (nodes, edges, Z) in (("isolated", _graph(W, 30, rng)), ("single edge", _graph(W, 2, rng))):
        if name == "isolated":
            edges, Z = edges[edges.max(1) < 29], Z[edges.max(1) < 29]
        prob = _problem(W, nodes, edges, Z, dt)
        Mn, _, Hd, g = _linearize(prob, W)
        s = NodeSystem(W, Mn, prob.nother, prob.nptr, Hd, g, scale, dmin, dmax)
        _, x, st, _, _ = _solve(s, tol, maxiter, [8])
        assert st[CG_DONE] == 1.0 and 0 < st[CG_ITERS] < maxiter and torch.isfinite(st).all(), (name, st.tolist())
        assert torch.isfinite(x).all()
        if name == "isolated":
            clamp = torch.tensor(dmin, dtype=dt) * torch.tensor(scale, dtype=dt)
            assert torch.equal(s.Hdamp[29].cpu(), torch.from_numpy(np.diag(np.full(W, clamp.item()))[np.triu_indices(W)]).to(dt))
            assert torch.equal(s.extra[29].cpu(), clamp.expand(W)) and torch.count_nonzero(x[29]) == 0
        H = _sparse_H(_np(Hd), _np(Mn), prob.nptr.cpu().numpy(), prob.nother.cpu().numpy(), W)
        A, gv = _damped(H, scale, dmin, dmax), _np(g).reshape(-1)
        _check_pcg(f"W={W} {dtn} {name} iters={int(st[CG_ITERS])}", H, A, gv, _np(x).reshape(-1),
                   spla.spsolve(A.tocsc(), -gv), scale, tol, dt, 1e-8)


# --------------------------------------------------------------------------------------- B. BAL reduced-camera PCG, W = 9
def _bal_system(C, dt):
    d = B.problem(7, C=C, P=2 * C, M=8 * C)
    lay = Layout(d, dt)
    K, T, P = cu(d["K0"], dt), cu(d["T0"], dt), cu(d["P0"], dt)
    Y4s, rs, Hcc, Hpp, gc, gp, _ = _fused.bal_linearize(K, T, P, lay.pix, lay.pidx, lay.geom)
    return lay, K, T, Y4s, rs, Hcc, Hpp, gc, gp


# C <= 2048: cg_vec_small_kernel<256>; 2048 < C <= 4096: cg_vec_small_kernel<512>; C > 4096: cg_dot / cg_update / cg_dir
@pytest.mark.parametrize("C", [2048, 2049, 4096, 4097])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_bal_pcg_chunks_and_stop_reasons(dtn, C):
    """b200_lm_bal_pcg on both edges of both single-CTA kernels and the grid path: chunk invariance (bit-identical to
    _fused.bal_solve) and every stop reason of the guard, with -Hc as the block-diagonal part for breakdown."""
    dt = PCG_DT[dtn][0]
    tol = 1e-10 if dt == torch.float64 else 1e-5
    lay, K, T, Y4s, rs, Hcc, Hpp, gc, gp = _bal_system(C, dt)
    kernel = "cg_vec_small_kernel<256>" if C <= 2048 else "cg_vec_small_kernel<512>" if C <= 4096 else \
        f"grid path, {min(_cdiv(C, THREADS), _cap())} CTAs"
    tag = f"BAL {dtn} C={C} {kernel}"
    make = lambda scale, negate=False: BalSystem(lay, K, T, Y4s, Hcc, Hpp, gc, gp, scale, negate=negate)
    _, x, st, _, _ = _chunk_invariance(lambda: make(1.5), tol, 2000, tag)
    xc, _, iters, _ = _fused.bal_solve(Y4s, K, T, rs, lay.cidx, lay.pidx, lay.geom, Hcc, Hpp, gc, gp, 1.5, 1e-6, 1e32, tol, 2000)
    assert torch.equal(xc, x) and iters == int(st[CG_ITERS].item()), tag
    _stop_reasons(make, lambda scale: make(scale, negate=True), None, tag, 1e-4 if dt == torch.float64 else 1e-3)


# ----------------------------------------------------------------- C. one-call trial against the Python-driven trial
def _trial_problem(family, scenario, dt):
    """(model, input, LM keyword arguments, steps, step at which the caller's loss is halved or None)."""
    W = {"se3": 6, "sim3": 7, "so3": 3}[family]
    lt = GROUPS[W][3]
    if family == "sim3" and scenario == "reject":         # the far start of the golden runs: rejected trials of its own
        import os
        g = np.load(os.path.join(os.path.dirname(__file__), "golden", "sim3pgo.npz"))
        nodes, edges, Z, steps = g["reject/nodes0"], g["reject/edges"], g["reject/Z"], len(g["reject/loss"])
        forced = None
    else:
        nodes, edges, Z = _graph(W, 300, np.random.default_rng(70 + W), loops=600, noise=0.3)
        steps, forced = 5, (2 if scenario == "reject" else None)
    if scenario == "maxiter":
        kw = dict(strategy=pp.optim.strategy.Constant(damping=1e-4), solver=PCG(tol=1e-30, maxiter=13))
    else:
        kw = dict(strategy=pp.optim.strategy.TrustRegion(), solver=PCG(tol=1e-13 if dt == torch.float64 else 1e-6))
    model = pp.module.PoseGraph(lt(cu(nodes, dt)))
    return model, (torch.from_numpy(edges).cuda(), lt(cu(Z, dt))), dict(kw, sparse=True, reject=4), steps, forced


def _run_lm(family, scenario, dt, device, monkeypatch):
    """Per step: loss, nodes, reject_count, cg_iters; per trial: (retry, cur, trial loss, predicted, cg_iters, status).
    On the one-call route every rejected trial leaves the nodes as they were, and a retried trial leaves the
    linearisation (Mn) as it was and never runs the linearisation kernel (its per-slot gradients `un`, filled with NaN
    before the trial, are still NaN after it)."""
    model, inp, kw, steps, forced = _trial_problem(family, scenario, dt)
    trials = []
    with monkeypatch.context() as m:
        if device:
            orig = structured.PGOProblem.device_trial

            def device_trial(self, ds, scale, dmin, dmax, retry):
                before, Mn = self._nodes().clone(), ds.buf["Mn"].clone()
                if retry:
                    ds.buf["un"].fill_(float("nan"))
                st = orig(self, ds, scale, dmin, dmax, retry)
                status = st[_lmstep.ST_STATUS]
                if status == 0.0:
                    assert torch.equal(self._nodes(), before), "a rejected trial changed the nodes"
                if retry:
                    assert torch.equal(ds.buf["Mn"], Mn), "a retried trial changed the linearisation"
                    assert torch.isnan(ds.buf["un"]).all(), "a retried trial ran the linearisation"
                trials.append((retry, st[_lmstep.ST_CUR], st[_lmstep.ST_TRIAL], st[_lmstep.ST_PRED], self.cg_iters, status))
                return st
            m.setattr(structured.PGOProblem, "device_trial", device_trial)
        else:
            m.setattr(structured.PGOProblem, "device_step", lambda self, s: None)
            orig = structured.PGOProblem.trial

            def trial(self, lin, scale, dmin, dmax):
                r = orig(self, lin, scale, dmin, dmax)
                # host decision of optimizer.py (status filled in below from the reject count)
                trials.append([None, r["cur"], r["loss"], r["predicted"], self.cg_iters, None])
                return r
            m.setattr(structured.PGOProblem, "trial", trial)
        opt = pp.optim.LM(model, **kw)
        out = []
        for k in range(steps):
            if k == forced:                  # a loss set by the caller below what any trial reaches: every trial is rejected
                opt.loss = opt.loss * 0.5     # up to LM(reject=...), then the last one is accepted
            n0 = len(trials)
            loss = float(opt.step(input=inp))
            prob = opt._problem
            assert (getattr(prob, "_pds", None) is not None) == device
            if not device:                   # trials n0.. of this step: rejected but the last (optimizer.py:314-319)
                for i in range(n0, len(trials)):
                    trials[i][0] = i > n0
                    trials[i][5] = 1.0 if i == len(trials) - 1 else 0.0
                    trials[i] = tuple(trials[i])
            out.append((loss, model.nodes.detach().tensor().clone(), opt.reject_count, prob.cg_iters))
    return out, trials


@pytest.mark.parametrize("scenario", ["reject", "maxiter"])
@pytest.mark.parametrize("family", ["so3", "sim3", "se3"])
@pytest.mark.parametrize("dtn", ["f64", "f32"])
def test_one_call_trial_matches_python_trial_bit_for_bit(dtn, family, scenario, monkeypatch):
    """b200_lm_pgo2_step (families 3, 2 and 0) enqueues the entry points of the Python-driven trial in the same chunks
    (hint, then 8), and neither route uses atomics: losses, nodes, reject counts, CG iteration counts, predicted
    reductions and decisions agree bit for bit.  'reject': runs with rejected (and retried) trials; 'maxiter':
    PCG(maxiter=13), not a multiple of the chunk size, with a hint (14) larger than it."""
    dt = PCG_DT[dtn][0]
    dev, dev_trials = _run_lm(family, scenario, dt, True, monkeypatch)
    host, host_trials = _run_lm(family, scenario, dt, False, monkeypatch)
    tag = f"{family} {scenario} {dtn}"
    for k, (a, b) in enumerate(zip(dev, host)):
        assert a[0] == b[0] and a[2] == b[2] and a[3] == b[3], (tag, k, a[0], b[0], a[2:], b[2:])
        assert torch.equal(a[1], b[1]), (tag, k, "nodes")
    assert dev_trials == host_trials, (tag, dev_trials, host_trials)
    rejects = [s[2] for s in dev]
    if scenario == "reject":
        assert sum(rejects) > 0 and any(t[0] for t in dev_trials), (tag, rejects)
    else:
        assert all(t[4] == 13 for t in dev_trials), (tag, [t[4] for t in dev_trials])
    print(tag, f"{len(dev_trials)} trials, rejects per step {rejects}, CG iterations {[t[4] for t in dev_trials]}")
