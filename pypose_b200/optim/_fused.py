"""torch custom ops `b200pose::lm_*` over the fused LM kernels (csrc/lm.cu).

Like the Lie ops, only the CUDA dispatch key has a kernel.  All host-visible scalars come back as
a small fp64 tensor on the device (`sums`), so the caller decides when to synchronise.
"""
import ctypes
from typing import NamedTuple

import torch
from torch import Tensor

from .. import _C

NS = "b200pose"
_ws = {}


_WS_SLOTS = 4


def _workspaces(device):
    """Per-device fp64 reduction workspaces (_WS_SLOTS, doubles), zeroed once (the kernels re-arm them).  Kernels of one
    LM trial that the host reads together use different slots, so their totals sit at [k, 0:4] and ONE strided copy
    brings them to the host."""
    key = (device.type, device.index)
    w = _ws.get(key)
    if w is None:
        n = _C.lib().b200_lm_workspace_doubles
        n.restype = ctypes.c_longlong
        w = torch.zeros(_WS_SLOTS, int(n()), dtype=torch.float64, device=device)
        _ws[key] = w
    return w


def _workspace(device):
    return _workspaces(device)[0]


def _p(t):
    return t.data_ptr() if t is not None else None        # c_void_p argtypes take ints / None


def _launch(base, ref: Tensor, args, n):
    if not ref.is_cuda:
        raise _C.B200PoseError(f"{base}: expected CUDA tensors (no CPU path), got {ref.device}")
    _C.enqueue(base + ("_f32" if ref.dtype is torch.float32 else "_" + _C.suffix(ref.dtype)), ref, *args, n)


def _same(*ts):
    dt, dev = ts[0].dtype, ts[0].device
    for t in ts:
        if t.dtype != dt or t.device != dev:
            raise TypeError(f"b200pose LM ops need one dtype/device for all floating inputs (got {t.dtype} on {t.device}, "
                            f"expected {dt} on {dev})")
    return [t.contiguous() for t in ts]


torch.library.define(f"{NS}::lm_poseinv_loss", "(Tensor P, Tensor X, int robust, float delta) -> Tensor")
torch.library.define(f"{NS}::lm_poseinv_trial",
                     "(Tensor P, Tensor X, float scale, float dmin, float dmax, int robust, float delta) -> (Tensor, Tensor)")
torch.library.define(f"{NS}::lm_reproj_accum",
                     "(Tensor poses, Tensor pts, Tensor pix, Tensor seg, int robust, float delta) -> (Tensor, Tensor, Tensor)")
torch.library.define(f"{NS}::lm_solve6_retract",
                     "(Tensor H, Tensor g, Tensor P, float scale, float dmin, float dmax) -> (Tensor, Tensor, Tensor)")
torch.library.define(f"{NS}::lm_reproj_loss",
                     "(Tensor poses, Tensor pts, Tensor pix, Tensor seg, int robust, float delta) -> Tensor")
torch.library.define(f"{NS}::lm_reproj_residual", "(Tensor poses, Tensor pts, Tensor pix, Tensor cidx) -> Tensor")


torch.library.define(f"{NS}::lm_pgo_linearize",
                     "(Tensor nodes, Tensor Z, Tensor ei, Tensor ej, int robust, float delta) -> (Tensor, Tensor, Tensor)")
torch.library.define(f"{NS}::lm_pgo_linearize_w",
                     "(Tensor nodes, Tensor Z, Tensor ei, Tensor ej, Tensor W, int robust, float delta) -> "
                     "(Tensor, Tensor, Tensor, Tensor, Tensor)")
torch.library.define(f"{NS}::lm_pgo_scatter", "(Tensor M, Tensor u, Tensor ei, Tensor ej, int n) -> (Tensor, Tensor)")
torch.library.define(f"{NS}::lm_pgo_spmv", "(Tensor M, Tensor ei, Tensor ej, Tensor x, Tensor y0) -> Tensor")
torch.library.define(f"{NS}::lm_pgo_loss", "(Tensor nodes, Tensor Z, Tensor ei, Tensor ej, int robust, float delta) -> Tensor")


def _pgo_linearize(nodes, Z, ei, ej, robust=0, delta=1.0):
    nodes, Z = _same(nodes, Z)
    E = Z.shape[0]
    ws = _workspace(nodes.device)
    M = torch.empty(E, 21, dtype=nodes.dtype, device=nodes.device)
    u = torch.empty(E, 6, dtype=nodes.dtype, device=nodes.device)
    _launch("b200_lm_pgo_linearize", nodes, [_p(nodes), _p(Z), _p(ei), _p(ej), _p(M), _p(u), _p(ws), int(robust),
                                             float(delta)], E)
    return M, u, ws[:1].clone()


def _pgo_linearize_w(nodes, Z, ei, ej, W, robust=0, delta=1.0):
    """W: (E,6,6) or (1,6,6) symmetric information matrices -> weighted (M, u), unweighted (M0, u0), cost."""
    nodes, Z, W = _same(nodes, Z, W)
    E = Z.shape[0]
    ws = _workspace(nodes.device)
    M, M0 = (torch.empty(E, 21, dtype=nodes.dtype, device=nodes.device) for _ in range(2))
    u, u0 = (torch.empty(E, 6, dtype=nodes.dtype, device=nodes.device) for _ in range(2))
    _launch("b200_lm_pgo_linearize_w", nodes, [_p(nodes), _p(Z), _p(ei), _p(ej), _p(W), 36 if W.shape[0] == E and E > 1 else 0,
                                               _p(M), _p(u), _p(M0), _p(u0), _p(ws), int(robust), float(delta)], E)
    return M, u, M0, u0, ws[:1].clone()


def _pgo_scatter(M, u, ei, ej, n):
    Hd = torch.zeros(n, 21, dtype=M.dtype, device=M.device)
    g = torch.zeros(n, 6, dtype=M.dtype, device=M.device)
    _launch("b200_lm_pgo_scatter", M, [_p(M), _p(u), _p(ei), _p(ej), _p(Hd), _p(g)], M.shape[0])
    return Hd, g


def _pgo_spmv(M, ei, ej, x, y0):
    """returns y0 + H x."""
    y = y0.clone()
    x = x.contiguous()
    _launch("b200_lm_pgo_spmv", M, [_p(M), _p(ei), _p(ej), _p(x), _p(y)], M.shape[0])
    return y


def _pgo_loss(nodes, Z, ei, ej, robust=0, delta=1.0):
    nodes, Z = _same(nodes, Z)
    ws = _workspace(nodes.device)
    _launch("b200_lm_pgo_loss", nodes, [_p(nodes), _p(Z), _p(ei), _p(ej), _p(ws), int(robust), float(delta)], Z.shape[0])
    return ws[:1].clone()


torch.library.define(f"{NS}::lm_ba_linearize",
                     "(Tensor poses, Tensor points, Tensor pix, Tensor cidx, Tensor pidx, int robust, float delta) -> "
                     "(Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)")
torch.library.define(f"{NS}::lm_ba_wtx", "(Tensor Jc, Tensor Jp, Tensor cidx, Tensor pidx, Tensor x, int npts) -> Tensor")
torch.library.define(f"{NS}::lm_ba_wv", "(Tensor Jc, Tensor Jp, Tensor cidx, Tensor pidx, Tensor v, int ncam) -> Tensor")
torch.library.define(f"{NS}::lm_ba_loss",
                     "(Tensor poses, Tensor points, Tensor pix, Tensor cidx, Tensor pidx, int robust, float delta) -> Tensor")


def _ba_linearize(poses, points, pix, cidx, pidx, robust=0, delta=1.0):
    poses, points, pix = _same(poses, points, pix)
    m, C, P = pix.shape[0], poses.shape[0], points.shape[0]
    dt, dev = poses.dtype, poses.device
    ws = _workspace(dev)
    Jc, Jp, rs = (torch.empty(m, w, dtype=dt, device=dev) for w in (12, 6, 2))
    Hcc, Hpp = torch.zeros(C, 21, dtype=dt, device=dev), torch.zeros(P, 6, dtype=dt, device=dev)
    gc, gp = torch.zeros(C, 6, dtype=dt, device=dev), torch.zeros(P, 3, dtype=dt, device=dev)
    _launch("b200_lm_ba_linearize", poses, [_p(poses), _p(points), _p(pix), _p(cidx), _p(pidx), _p(Jc), _p(Jp), _p(rs),
                                            _p(Hcc), _p(Hpp), _p(gc), _p(gp), _p(ws), int(robust), float(delta)], m)
    return Jc, Jp, rs, Hcc, Hpp, gc, gp, ws[:1].clone()


def _ba_wtx(Jc, Jp, cidx, pidx, x, npts):
    t = torch.zeros(npts, 3, dtype=Jc.dtype, device=Jc.device)
    x = x.contiguous()
    _launch("b200_lm_ba_wtx", Jc, [_p(Jc), _p(Jp), _p(cidx), _p(pidx), _p(x), _p(t)], Jc.shape[0])
    return t


def _ba_wv(Jc, Jp, cidx, pidx, v, ncam):
    y = torch.zeros(ncam, 6, dtype=Jc.dtype, device=Jc.device)
    v = v.contiguous()
    _launch("b200_lm_ba_wv", Jc, [_p(Jc), _p(Jp), _p(cidx), _p(pidx), _p(v), _p(y)], Jc.shape[0])
    return y


def _ba_loss(poses, points, pix, cidx, pidx, robust=0, delta=1.0):
    poses, points, pix = _same(poses, points, pix)
    ws = _workspace(poses.device)
    _launch("b200_lm_ba_loss", poses, [_p(poses), _p(points), _p(pix), _p(cidx), _p(pidx), _p(ws), int(robust),
                                       float(delta)], pix.shape[0])
    return ws[:1].clone()


def _poseinv_loss(P, X, robust=0, delta=1.0):
    P, X = _same(P, X)
    ws = _workspace(P.device)
    _launch("b200_lm_poseinv_loss", P, [_p(P), _p(X), _p(ws), int(robust), float(delta)], P.shape[0])
    return ws[:1].clone()


def _poseinv_trial(P, X, scale, dmin, dmax, robust=0, delta=1.0):
    P, X = _same(P, X)
    ws = _workspace(P.device)
    Pt = torch.empty_like(P)
    _launch("b200_lm_poseinv_trial", P, [_p(P), _p(X), _p(Pt), _p(ws), scale, dmin, dmax, int(robust), float(delta)],
            P.shape[0])
    return Pt, ws[:4].clone()


def _reproj_accum(poses, pts, pix, seg, robust=0, delta=1.0):
    poses, pts, pix = _same(poses, pts, pix)
    assert seg.dtype == torch.int32 and seg.numel() == poses.shape[0] + 1
    ws = _workspace(poses.device)
    C = poses.shape[0]
    H = torch.empty(C, 21, dtype=poses.dtype, device=poses.device)
    g = torch.empty(C, 6, dtype=poses.dtype, device=poses.device)
    _launch("b200_lm_reproj_accum", poses, [_p(poses), _p(pts), _p(pix), _p(seg), _p(H), _p(g), _p(ws), int(robust),
                                                   float(delta)], C)
    return H, g, ws[:1].clone()


def _solve6_retract(H, g, P, scale, dmin, dmax):
    H, g, P = _same(H, g, P)
    ws = _workspace(P.device)
    Pt, D = torch.empty_like(P), torch.empty(P.shape[0], 6, dtype=P.dtype, device=P.device)
    _launch("b200_lm_solve6_retract", P, [_p(H), _p(g), _p(P), _p(Pt), _p(D), _p(ws), scale, dmin, dmax], P.shape[0])
    return Pt, D, ws[:2].clone()


def _reproj_loss(poses, pts, pix, seg, robust=0, delta=1.0):
    poses, pts, pix = _same(poses, pts, pix)
    assert seg.dtype == torch.int32 and seg.numel() == poses.shape[0] + 1
    ws = _workspace(poses.device)
    _launch("b200_lm_reproj_loss", poses, [_p(poses), _p(pts), _p(pix), _p(seg), _p(ws), int(robust), float(delta)],
            poses.shape[0])
    return ws[:1].clone()


def _reproj_residual(poses, pts, pix, cidx):
    poses, pts, pix = _same(poses, pts, pix)
    assert cidx.dtype == torch.int32
    r = torch.empty(pts.shape[0], 2, dtype=poses.dtype, device=poses.device)
    _launch("b200_lm_reproj_residual", poses, [_p(poses), _p(pts), _p(pix), _p(cidx), _p(r)], pts.shape[0])
    return r


torch.library.define(f"{NS}::lm_reproj2_accum",
                     "(Tensor nodes, Tensor pts, Tensor pix, Tensor pseg, Tensor pa, Tensor pb, float[] intr, int robust, "
                     "float delta) -> (Tensor, Tensor, Tensor)")
torch.library.define(f"{NS}::lm_reproj2_loss",
                     "(Tensor nodes, Tensor pts, Tensor pix, Tensor pseg, Tensor pa, Tensor pb, float[] intr, int robust, "
                     "float delta) -> Tensor")


def _intr(intr):
    return ctypes.addressof((ctypes.c_double * 5)(*[float(v) for v in intr]))


def _reproj2_accum(nodes, pts, pix, pseg, pa, pb, intr, robust=0, delta=1.0):
    nodes, pts, pix = _same(nodes, pts, pix)
    E = pa.shape[0]
    ws = _workspace(nodes.device)
    M = torch.empty(E, 21, dtype=nodes.dtype, device=nodes.device)
    u = torch.empty(E, 6, dtype=nodes.dtype, device=nodes.device)
    k = (ctypes.c_double * 5)(*[float(v) for v in intr])
    _launch("b200_lm_reproj2_accum", nodes, [_p(nodes), _p(pts), _p(pix), _p(pseg), _p(pa), _p(pb), ctypes.addressof(k), _p(M),
                                             _p(u), _p(ws), int(robust), float(delta)], E)
    return M, u, ws[:1].clone()


def _reproj2_loss(nodes, pts, pix, pseg, pa, pb, intr, robust=0, delta=1.0):
    nodes, pts, pix = _same(nodes, pts, pix)
    ws = _workspace(nodes.device)
    k = (ctypes.c_double * 5)(*[float(v) for v in intr])
    _launch("b200_lm_reproj2_loss", nodes, [_p(nodes), _p(pts), _p(pix), _p(pseg), _p(pa), _p(pb), ctypes.addressof(k), _p(ws),
                                            int(robust), float(delta)], pa.shape[0])
    return ws[:1].clone()


torch.library.impl(f"{NS}::lm_reproj2_accum", "CUDA")(_reproj2_accum)
torch.library.impl(f"{NS}::lm_reproj2_loss", "CUDA")(_reproj2_loss)
torch.library.impl(f"{NS}::lm_ba_linearize", "CUDA")(_ba_linearize)
torch.library.impl(f"{NS}::lm_ba_wtx", "CUDA")(_ba_wtx)
torch.library.impl(f"{NS}::lm_ba_wv", "CUDA")(_ba_wv)
torch.library.impl(f"{NS}::lm_ba_loss", "CUDA")(_ba_loss)
torch.library.impl(f"{NS}::lm_pgo_linearize", "CUDA")(_pgo_linearize)
torch.library.impl(f"{NS}::lm_pgo_linearize_w", "CUDA")(_pgo_linearize_w)
torch.library.impl(f"{NS}::lm_pgo_scatter", "CUDA")(_pgo_scatter)
torch.library.impl(f"{NS}::lm_pgo_spmv", "CUDA")(_pgo_spmv)
torch.library.impl(f"{NS}::lm_pgo_loss", "CUDA")(_pgo_loss)
torch.library.impl(f"{NS}::lm_poseinv_loss", "CUDA")(_poseinv_loss)
torch.library.impl(f"{NS}::lm_poseinv_trial", "CUDA")(_poseinv_trial)
torch.library.impl(f"{NS}::lm_reproj_accum", "CUDA")(_reproj_accum)
torch.library.impl(f"{NS}::lm_solve6_retract", "CUDA")(_solve6_retract)
torch.library.impl(f"{NS}::lm_reproj_loss", "CUDA")(_reproj_loss)
torch.library.impl(f"{NS}::lm_reproj_residual", "CUDA")(_reproj_residual)


# ----------------------------------------------------------------------------------------------------
# Fast path used by optim/structured.py: for CUDA tensors call the C-ABI directly (the torch dispatcher
# plus a Python kernel costs ~20-40 us per op, comparable to the kernels themselves); CPU tensors go
# through torch.ops so that the test-only oracle kernels are reachable.
# ----------------------------------------------------------------------------------------------------
def call(name, *args):
    first = args[0]
    if first.is_cuda:
        return _DIRECT[name](*args)
    return getattr(torch.ops.b200pose, name)(*args)


_DIRECT = {"lm_poseinv_loss": _poseinv_loss, "lm_poseinv_trial": _poseinv_trial, "lm_reproj_accum": _reproj_accum,
           "lm_solve6_retract": _solve6_retract, "lm_reproj_loss": _reproj_loss, "lm_reproj_residual": _reproj_residual,
           "lm_pgo_linearize": _pgo_linearize, "lm_pgo_linearize_w": _pgo_linearize_w, "lm_pgo_scatter": _pgo_scatter, "lm_pgo_spmv": _pgo_spmv,
           "lm_pgo_loss": _pgo_loss, "lm_ba_linearize": _ba_linearize, "lm_ba_wtx": _ba_wtx, "lm_ba_wv": _ba_wv,
           "lm_ba_loss": _ba_loss, "lm_reproj2_accum": _reproj2_accum, "lm_reproj2_loss": _reproj2_loss}

LM_OPS = ["lm_poseinv_loss", "lm_poseinv_trial", "lm_reproj_accum", "lm_solve6_retract", "lm_reproj_loss",
          "lm_reproj_residual"]
ops = torch.ops.b200pose


# ----------------------------------------------------------------------------------------------------
# Device-resident PCG (csrc/pcg.cu), CUDA only and single-rank only: the multi-rank route all-reduces every
# operator product on the host side (optim/structured.py:_pcg).
# ----------------------------------------------------------------------------------------------------
CG_CHUNK = 8            # iterations enqueued per host call / per read of the done flag
_cg_state = {}


def _cg(device):
    key = (device.type, device.index)
    s = _cg_state.get(key)
    if s is None:
        s = _cg_state[key] = torch.zeros(16, dtype=torch.float64, device=device)
    return s


def _run_chunks(enqueue, cg, maxiter, hint=0):
    """enqueue(first_iter, iters) until the device reports done; returns the iteration count.  `hint` (the iteration
    count of the previous solve of this problem) sizes the first chunk: consecutive LM trials need about the same
    number of iterations, so most solves cost exactly one host read."""
    it = 0
    while True:
        n = max(1, min(hint if (it == 0 and hint > 0) else CG_CHUNK, maxiter - it))
        enqueue(it, n)
        it += n
        st = cg.tolist()                                  # the one host sync per chunk
        if st[5] != 0.0 or it >= maxiter:
            return int(st[6])


class NodeWidth(NamedTuple):
    """One block width W of the node-ordered route (csrc/pcg2.cu Slot<W>): words per slot, packed words of a W x W block,
    parameter width D of a node and the width-specific entry points."""
    slot: int
    packed: int
    D: int
    node_sums: str
    damp_inv: str
    pcg: str
    cg_finish: str
    predicted: str


# W = 6: SE3 pose graphs and pose pairs; 7: Sim3 pose graphs; 3: SO3 pose graphs (include/b200pose.h, b200_pgo_step_args)
NODE_WIDTHS = {
    6: NodeWidth(24, 21, 7, "b200_lm_pgo2_node_sums", "b200_lm_blk6_damp_inv", "b200_lm_pgo2_pcg", "b200_lm_cg_finish",
                 "b200_lm_pgo2_predicted"),
    7: NodeWidth(28, 28, 8, "b200_lm_sim3pgo_node_sums", "b200_lm_sim3pgo_damp_inv", "b200_lm_sim3pgo_pcg",
                 "b200_lm_sim3pgo_cg_finish", "b200_lm_sim3pgo_predicted"),
    3: NodeWidth(8, 6, 4, "b200_lm_so3pgo_node_sums", "b200_lm_so3pgo_damp_inv", "b200_lm_so3pgo_pcg",
                 "b200_lm_so3pgo_cg_finish", "b200_lm_so3pgo_predicted"),
}
# block width and node-ordered linearisation of each problem kind with edges (ei, ej, Z); "reproj2" is linearised by pose pair
KIND_WIDTH = {"pgo": 6, "reproj2": 6, "sim3": 7, "so3": 3}
_EDGE_LINEARIZE = {"pgo": "b200_lm_pgo_linearize_n", "sim3": "b200_lm_sim3pgo_linearize", "so3": "b200_lm_so3pgo_linearize"}


def pgo_linearize_nodes(kind, prob, nodes, robust, delta):
    """Blocks of the current linearisation directly in node order (csrc/lm.cu store_edge_blocks, csrc/sim3pgo.cu,
    csrc/so3pgo.cu) and, by gather, the diagonal blocks Hd and J^T R.  kind: "pgo" (Log(Z^-1 A^-1 B) edges), "reproj2"
    (pose pairs), "sim3" or "so3" (Log(Z^-1 A^-1 B) on Sim3 / SO3 nodes); its block width is KIND_WIDTH[kind]."""
    E, N = prob.ei.shape[0], prob.nptr.shape[0] - 1
    E2 = 2 * E
    dt, dev = nodes.dtype, nodes.device
    ws = _workspace(dev)
    W = KIND_WIDTH[kind]
    spec = NODE_WIDTHS[W]
    Mn, un = torch.empty(E2, spec.slot, dtype=dt, device=dev), torch.empty(E2, W, dtype=dt, device=dev)
    if kind == "reproj2":
        k = (ctypes.c_double * 5)(*prob.intr)
        _launch("b200_lm_reproj2_accum_n", nodes, [_p(nodes), _p(prob.pts), _p(prob.pix), _p(prob.pseg), _p(prob.pa), _p(prob.pb),
                                                   ctypes.addressof(k), _p(prob.epos_i), _p(prob.epos_j), _p(Mn), _p(un), _p(ws),
                                                   int(robust), float(delta)], E)
    else:
        _launch(_EDGE_LINEARIZE[kind], nodes, [_p(nodes), _p(prob.Z), _p(prob.ei), _p(prob.ej), _p(prob.epos_i), _p(prob.epos_j),
                                               _p(Mn), _p(un), _p(ws), int(robust), float(delta)], E)
    cur = ws[:1].clone()
    Hd, g = torch.empty(N, spec.packed, dtype=dt, device=dev), torch.empty(N, W, dtype=dt, device=dev)
    _launch(spec.node_sums, nodes, [_p(Mn), _p(un), _p(prob.nptr), _p(Hd), _p(g)], N)
    return Mn, Hd, g, cur


def pgo_solve_nodes(Mn, nother, nptr, Hd, g, scale, dmin, dmax, tol, maxiter, hint=0):
    """(H + clamp/damping) x = -g on node-ordered blocks (csrc/pcg2.cu): two launches per iteration, no atomics.
    The block width W (NODE_WIDTHS) is g's.  Returns x (n,W), iterations, predicted (1,) fp64 on device."""
    dev, dt, n, W = Mn.device, Mn.dtype, Hd.shape[0], g.shape[1]
    spec = NODE_WIDTHS[W]
    ws, cg = _workspace(dev), _cg(dev)
    extra = torch.empty(n, W, dtype=dt, device=dev)
    Minv = torch.empty_like(Hd)
    x, r, z, p0, p1, q, xbest = (torch.empty(n, W, dtype=dt, device=dev) for _ in range(7))
    maxiter = int(maxiter) if maxiter is not None else 10 * W * n
    _launch(spec.damp_inv, Mn, [_p(Hd), float(scale), float(dmin), float(dmax), _p(None), _p(extra), _p(Minv)], n)
    iters = _run_chunks(lambda it0, k: _launch(spec.pcg, Mn, [
        _p(Mn), _p(nother), _p(nptr), _p(Minv), _p(extra), _p(g), _p(x), _p(r), _p(z), _p(p0), _p(p1), _p(q), _p(xbest),
        _p(cg), _p(ws), float(tol), maxiter, it0, k], n), cg, maxiter, hint)
    _launch(spec.cg_finish, Mn, [_p(x), _p(xbest), _p(cg)], n)
    _launch(spec.predicted, Mn, [_p(Mn), _p(nother), _p(nptr), _p(x), _p(g), _p(ws)], n)
    return x, iters, ws[:1].clone()


def sim3pgo_loss(nodes, Z, ei, ej, robust=0, delta=1.0):
    """(1,) fp64 device tensor: sum rho(|r|^2) of the Sim3 pose graph at the given (N,8) nodes."""
    nodes, Z = _same(nodes, Z)
    ws = _workspace(nodes.device)
    _launch("b200_lm_sim3pgo_loss", nodes, [_p(nodes), _p(Z), _p(ei), _p(ej), _p(ws), int(robust), float(delta)], Z.shape[0])
    return ws[:1].clone()


def so3pgo_loss(nodes, Z, ei, ej, robust=0, delta=1.0):
    """(1,) fp64 device tensor: sum rho(|r|^2) of the SO3 pose graph at the given (N,4) nodes."""
    nodes, Z = _same(nodes, Z)
    ws = _workspace(nodes.device)
    _launch("b200_lm_so3pgo_loss", nodes, [_p(nodes), _p(Z), _p(ei), _p(ej), _p(ws), int(robust), float(delta)], Z.shape[0])
    return ws[:1].clone()


_NOCOMM = [None, 0, 1, 0, 0, 0, None]


def pgo_solve(M, ei, ej, Hd, g, scale, dmin, dmax, tol, maxiter, hint=0, unweighted=None, comm=None):
    """(H + clamp/damping) x = -g by device PCG.  Returns x (n,6), iterations, predicted (1,) fp64 on device.
    `unweighted` = (M0, u0): per-edge blocks without the information matrices, for the predicted reduction.
    `node` = (Mn, nother, nptr): node-ordered blocks -> the H product is a gather (deterministic) instead of a scatter."""
    dev, dt, n, E = M.device, M.dtype, Hd.shape[0], M.shape[0]
    ws, cg = _workspace(dev), _cg(dev)
    extra = torch.empty(n, 6, dtype=dt, device=dev)
    Minv = torch.empty(n, 21, dtype=dt, device=dev)
    _launch("b200_lm_blk6_damp_inv", M, [_p(Hd), float(scale), float(dmin), float(dmax), _p(None), _p(extra), _p(Minv)], n)
    x, r, z, p, q, xbest = (torch.empty(n, 6, dtype=dt, device=dev) for _ in range(6))
    maxiter = int(maxiter) if maxiter is not None else 10 * 6 * n
    def chunk(it0, k):
        _launch("b200_lm_pgo_pcg", M, [
            _p(M), _p(ei), _p(ej), E, _p(Minv), _p(extra), _p(g), _p(x), _p(r), _p(z), _p(p), _p(q), _p(xbest), _p(cg),
            _p(ws), float(tol), maxiter, it0, k, *(comm.pcg_args() if comm is not None else _NOCOMM)], n)
        if comm is not None:
            comm.consumed(k)           # one device all-reduce of q per iteration
    iters = _run_chunks(chunk, cg, maxiter, hint)
    _launch("b200_lm_cg_finish", M, [_p(x), _p(xbest), _p(cg)], n)     # best iterate unless the solve converged
    if unweighted is None:
        _launch("b200_lm_pgo_predicted", M, [_p(M), _p(ei), _p(ej), E, _p(x), _p(g), _p(ws)], n)
    else:
        _launch("b200_lm_pgo_predicted_edge", M, [_p(unweighted[0]), _p(unweighted[1]), _p(ei), _p(ej), _p(x), _p(ws)], E)
    return x, iters, ws[:1].clone()


def ba_linearize_det(poses, points, pix, pidx, geom, robust=0, delta=1.0):
    """Deterministic BA linearisation (csrc/ba.cu): Y4 / Y4p / rs per observation, camera blocks with one writer per camera,
    point blocks by gather.  `geom` = (cseg, split, tpi, ppos, cidx_p, pptr, pix_p) from BAProblem."""
    cseg, split, tpi, ppos, cidx_p, pptr, pix_p = geom
    poses, points, pix = _same(poses, points, pix)
    m, C, P = pix.shape[0], poses.shape[0], points.shape[0]
    dt, dev = poses.dtype, poses.device
    ws = _workspace(dev)
    Y4, Y4p, rs = (torch.empty(m, w, dtype=dt, device=dev) for w in (4, 4, 2))
    Hcc, gc = torch.empty(C, 21, dtype=dt, device=dev), torch.empty(C, 6, dtype=dt, device=dev)
    Hpp, gp = torch.empty(P, 6, dtype=dt, device=dev), torch.empty(P, 3, dtype=dt, device=dev)
    part = torch.empty(C * split, 27, dtype=dt, device=dev) if split > 1 else None
    _launch("b200_lm_ba_linearize_seg", poses, [_p(poses), _p(points), _p(pix), _p(pidx), _p(cseg), split, tpi, _p(Y4), _p(ppos),
                                                _p(Y4p), _p(rs), _p(Hcc), _p(gc), _p(part), _p(ws), int(robust), float(delta)], C)
    cur = ws[:1].clone()
    _launch("b200_lm_ba_point_blocks", poses, [_p(Y4p), _p(pix_p), _p(poses), _p(cidx_p), _p(pptr), _p(Hpp), _p(gp)], P)
    return (Y4, Y4p), rs, Hcc, Hpp, gc, gp, cur


def ba_solve(Y4s, poses, rs, cidx, pidx, geom, Hcc, Hpp, gc, gp, scale, dmin, dmax, tol, maxiter, hint=0, comm=None):
    """Schur-complement solve of the damped BA normal equations by device PCG; the Jacobian rows are rebuilt from
    Y4 (ba_linearize_det) and the poses it was linearised at.  No atomics: every camera / point sum has one writer.
    Returns xc (C,6), xp (P,3), iterations, predicted (1,) fp64 on device."""
    Y4, Y4p = Y4s                                         # camera-ordered and point-ordered rows
    cseg, split, tpi, _, cidx_p, pptr, _ = geom
    dev, dt = Y4.device, Y4.dtype
    m, C, P = Y4.shape[0], Hcc.shape[0], Hpp.shape[0]
    ws, cg = _workspace(dev), _cg(dev)
    Hc = torch.empty(C, 21, dtype=dt, device=dev)
    Hpinv = torch.empty(P, 6, dtype=dt, device=dev)
    Minv = torch.empty(C, 21, dtype=dt, device=dev)
    part = torch.empty(C * split, 21, dtype=dt, device=dev) if split > 1 else None
    seg = [_p(Y4), _p(poses), _p(pidx), _p(cseg), split, tpi]
    _launch("b200_lm_blk6_damp_inv", Y4, [_p(Hcc), float(scale), float(dmin), float(dmax), _p(Hc), _p(None), _p(None)], C)
    _launch("b200_lm_pt3_damp_inv", Y4, [_p(Hpp), float(scale), float(dmin), float(dmax), _p(Hpinv)], P)
    # multi-GPU: Hcc / Hpp / gc / gp are already reduced (replicated); every sum over observations below is a partial sum
    # of this rank's shard, the replicated term is contributed by rank 0 only, then one device all-reduce
    first = comm is None or comm.rank == 0
    Sd = Hc.clone() if first else torch.zeros_like(Hc)
    _launch("b200_lm_ba_schur_diag_seg", Y4, [*seg, _p(Hpinv), _p(Sd), _p(part)], C)
    bneg = gc.clone() if first else torch.zeros_like(gc)  # -(rhs) = gc - W Hpp^-1 gp
    _launch("b200_lm_ba_wv_seg", Y4, [*seg, _p(Hpinv), _p(gp), _p(bneg), _p(part)], C)
    if comm is not None:
        comm.sum_(Sd)
        comm.sum_(bneg)
    _launch("b200_lm_blk6_damp_inv", Y4, [_p(Sd), 1.0, -3.0e38, 3.0e38, _p(None), _p(None), _p(Minv)], C)
    x, r, z, p, q, xbest = (torch.empty(C, 6, dtype=dt, device=dev) for _ in range(6))
    t = torch.empty(P, 3, dtype=dt, device=dev)
    maxiter = int(maxiter) if maxiter is not None else 10 * 6 * C
    def chunk(it0, k):
        _launch("b200_lm_ba_pcg", Y4, [
            *seg, m, _p(Y4p), _p(cidx_p), _p(pptr), _p(Hc), _p(Hpinv), _p(Minv), _p(bneg), _p(x), _p(r), _p(z), _p(p), _p(q),
            _p(t), _p(part), _p(xbest), _p(cg), _p(ws), float(tol), maxiter, P, it0, k,
            *(comm.pcg_args() if comm is not None else _NOCOMM)], C)
        if comm is not None:
            comm.consumed(2 * k)           # W^T p and W t are reduced in every iteration
    iters = _run_chunks(chunk, cg, maxiter, hint)
    _launch("b200_lm_cg_finish", Y4, [_p(x), _p(xbest), _p(cg)], C)
    xp = torch.empty(P, 3, dtype=dt, device=dev)          # dp = -Hpp^-1 (gp + W^T dc)
    _launch("b200_lm_ba_wtx_gather", Y4, [_p(Y4p), _p(poses), _p(cidx_p), _p(pptr), _p(Hpinv), _p(x), _p(gp if first else None),
                                          -1.0, _p(xp)], P)
    if comm is not None:
        comm.sum_(xp)
    _launch("b200_lm_ba_predicted", Y4, [_p(Y4), _p(poses), _p(rs), _p(cidx), _p(pidx), _p(x), _p(xp), _p(ws)], m)
    return x, xp, iters, ws[:1].clone()


def bal_linearize(intr, poses, points, pix, pidx, geom, robust=0, delta=1.0):
    """BAL linearisation (csrc/bal.cu): Y4 / Y4p / rs per observation, 9x9 camera blocks Hcc (C,45) and gc (C,9) with one
    writer per camera, point blocks Hpp (P,6) and gp (P,3) by gather.  `geom` as for ba_linearize_det (BALProblem)."""
    cseg, split, tpi, ppos, cidx_p, pptr, pix_p = geom
    intr, poses, points, pix = _same(intr, poses, points, pix)
    m, C, P = pix.shape[0], poses.shape[0], points.shape[0]
    dt, dev = poses.dtype, poses.device
    ws = _workspace(dev)
    Y4, Y4p, rs = (torch.empty(m, w, dtype=dt, device=dev) for w in (4, 4, 2))
    Hcc, gc = torch.empty(C, 45, dtype=dt, device=dev), torch.empty(C, 9, dtype=dt, device=dev)
    Hpp, gp = torch.empty(P, 6, dtype=dt, device=dev), torch.empty(P, 3, dtype=dt, device=dev)
    part = torch.empty(C * split, 54, dtype=dt, device=dev) if split > 1 else None
    _launch("b200_lm_bal_linearize_seg", poses, [_p(poses), _p(intr), _p(points), _p(pix), _p(pidx), _p(cseg), split, tpi,
                                                 _p(Y4), _p(ppos), _p(Y4p), _p(rs), _p(Hcc), _p(gc), _p(part), _p(ws),
                                                 int(robust), float(delta)], C)
    cur = ws[:1].clone()
    _launch("b200_lm_bal_point_blocks", poses, [_p(Y4p), _p(pix_p), _p(poses), _p(intr), _p(cidx_p), _p(pptr), _p(Hpp),
                                                _p(gp)], P)
    return (Y4, Y4p), rs, Hcc, Hpp, gc, gp, cur


def bal_solve(Y4s, intr, poses, rs, cidx, pidx, geom, Hcc, Hpp, gc, gp, scale, dmin, dmax, tol, maxiter, hint=0):
    """Schur-complement solve of the damped BAL normal equations by device PCG over the 9 unknowns of every camera
    (csrc/bal.cu); rows are rebuilt from Y4 and the intrinsics / poses of the linearisation.  Returns xc (C,9) =
    [xi | df, dk1, dk2], xp (P,3), iterations, predicted (1,) fp64 on device."""
    Y4, Y4p = Y4s
    cseg, split, tpi, _, cidx_p, pptr, _ = geom
    dev, dt = Y4.device, Y4.dtype
    m, C, P = Y4.shape[0], Hcc.shape[0], Hpp.shape[0]
    ws, cg = _workspace(dev), _cg(dev)
    Hc, Minv = torch.empty(C, 45, dtype=dt, device=dev), torch.empty(C, 45, dtype=dt, device=dev)
    Hpinv = torch.empty(P, 6, dtype=dt, device=dev)
    part = torch.empty(C * split, 45, dtype=dt, device=dev) if split > 1 else None
    y4, tp, kp, pi_, cs = _p(Y4), _p(poses), _p(intr), _p(pidx), _p(cseg)
    _launch("b200_lm_bal_damp_inv", Y4, [_p(Hcc), float(scale), float(dmin), float(dmax), _p(Hc), _p(None)], C)
    _launch("b200_lm_pt3_damp_inv", Y4, [_p(Hpp), float(scale), float(dmin), float(dmax), _p(Hpinv)], P)
    Sd = Hc.clone()
    _launch("b200_lm_bal_schur_diag_seg", Y4, [y4, tp, kp, pi_, cs, split, tpi, _p(Hpinv), _p(Sd), _p(part)], C)
    bneg = gc.clone()                                     # -(rhs) = gc - W Hpp^-1 gp
    _launch("b200_lm_bal_wv_seg", Y4, [y4, tp, kp, pi_, cs, split, tpi, _p(Hpinv), _p(gp), _p(bneg), _p(part)], C)
    _launch("b200_lm_bal_damp_inv", Y4, [_p(Sd), 1.0, -3.0e38, 3.0e38, _p(None), _p(Minv)], C)
    x, r, z, p, q, xbest = (torch.empty(C, 9, dtype=dt, device=dev) for _ in range(6))
    t = torch.empty(P, 3, dtype=dt, device=dev)
    maxiter = int(maxiter) if maxiter is not None else 10 * 9 * C
    iters = _run_chunks(lambda it0, k: _launch("b200_lm_bal_pcg", Y4, [
        y4, tp, kp, pi_, cs, split, tpi, m, _p(Y4p), _p(cidx_p), _p(pptr), _p(Hc), _p(Hpinv), _p(Minv), _p(bneg), _p(x), _p(r), _p(z), _p(p), _p(q),
        _p(t), _p(part), _p(xbest), _p(cg), _p(ws), float(tol), maxiter, P, it0, k], C), cg, maxiter, hint)
    _launch("b200_lm_bal_cg_finish", Y4, [_p(x), _p(xbest), _p(cg)], C)     # best iterate unless the solve converged
    xp = torch.empty(P, 3, dtype=dt, device=dev)          # dp = -Hpp^-1 (gp + W^T dc)
    _launch("b200_lm_bal_wtx_gather", Y4, [_p(Y4p), _p(poses), _p(intr), _p(cidx_p), _p(pptr), _p(Hpinv), _p(x), _p(gp),
                                           -1.0, _p(xp)], P)
    _launch("b200_lm_bal_predicted", Y4, [_p(Y4), _p(poses), _p(intr), _p(rs), _p(cidx), _p(pidx), _p(x), _p(xp), _p(ws)], m)
    return x, xp, iters, ws[:1].clone()


def bal_loss(intr, poses, points, pix, cidx, pidx, robust=0, delta=1.0):
    """(1,) fp64 device tensor: sum rho(|r|^2) of the BAL model at the given parameters."""
    ws = _workspace(poses.device)
    _launch("b200_lm_bal_loss", poses, [_p(poses), _p(intr), _p(points), _p(pix), _p(cidx), _p(pidx), _p(ws), int(robust),
                                        float(delta)], pix.shape[0])
    return ws[:1].clone()


def bal_retract(intr, poses, points, xc, xp):
    """Trial parameters: (K + dK, Exp(xi) T, p + dp) from xc (C,9) = [xi | dK] and xp (P,3)."""
    Kt, Tt, pt = torch.empty_like(intr), torch.empty_like(poses), torch.empty_like(points)
    _launch("b200_lm_bal_retract", poses, [_p(poses), _p(intr), _p(points), _p(xc), _p(xp), _p(Tt), _p(Kt), _p(pt),
                                           poses.shape[0]], points.shape[0])
    return Kt, Tt, pt


# ----------------------------------------------------------------------------------------------------
# Reprojection LM trial with the fewest host operations (the step is host-bound: ~30 us of kernels, see
# tools/prof_lm_host.py): outputs are caller-owned buffers, the three kernels reduce into three workspace
# slots and one strided 4x4 copy returns [cur | trial loss | predicted, failed].
# ----------------------------------------------------------------------------------------------------
def reproj_linearize(poses, pts, pix, seg, robust, delta, H, g):
    W = _workspaces(poses.device)
    _launch("b200_lm_reproj_accum", poses, [poses.data_ptr(), pts.data_ptr(), pix.data_ptr(), seg.data_ptr(), H.data_ptr(),
                                            g.data_ptr(), W[0].data_ptr(), int(robust), float(delta)], poses.shape[0])


def reproj_trial(H, g, poses, pts, pix, seg, scale, dmin, dmax, robust, delta, Pt):
    """-> (16,) fp64 device tensor: [0] current loss (from reproj_linearize), [4] trial loss, [8] predicted, [9] failed."""
    W = _workspaces(poses.device)
    n = poses.shape[0]
    _launch("b200_lm_solve6_retract", poses, [H.data_ptr(), g.data_ptr(), poses.data_ptr(), Pt.data_ptr(), None, W[2].data_ptr(),
                                              float(scale), float(dmin), float(dmax)], n)
    _launch("b200_lm_reproj_loss", poses, [Pt.data_ptr(), pts.data_ptr(), pix.data_ptr(), seg.data_ptr(), W[1].data_ptr(),
                                           int(robust), float(delta)], n)
    return W[:, :4].reshape(-1)              # non-contiguous view -> reshape copies (one small kernel)
