"""Structured LM problems: residual families whose Jacobian blocks are known in closed form.

The reference builds an (R x 7N) dense Jacobian by vmapped autograd even when it is exactly
block-diagonal (SURVEY.md §3.2-3.3).  For the families below the same normal equations are formed
block-wise inside fused kernels (csrc/lm.cu, lm_math.cuh):

  PoseInv  — README.md:120-129 InvNet:  forward(input) = (pose @ input).Log().tensor()
  Reproj   — README.md:170-178 project / SURVEY.md §8d cfg 5-min:  -(T_c p)[:2]/(T_c p)[2] - z

PoseInv is *recognised* from an unchanged user module by recording the LieTensor ops its forward
executes (one group multiply followed by one Log).  Reproj is recognised by model type
(pypose_b200.module.PoseReproj).

Multi-GPU (`group`): PoseInv shards poses (each rank owns its rows; only the scalar sums are
all-reduced).  Reproj shards residuals (each rank accumulates H/g for its rows; H, g and the
scalars are all-reduced; the 6x6 solves run redundantly on every rank).
"""
import torch

from .. import _C
from ..lietensor import lietensor as _lt
from ..lietensor.lietensor import LieTensor, Parameter, SE3_type, SO3_type, Sim3_type
from ..lietensor.scan import _sms
from . import _fused  # noqa: F401  (registers the ops)
from . import _lmstep

ops = torch.ops.b200pose


def _allreduce(t, group):
    if group is not None and torch.distributed.is_available() and torch.distributed.is_initialized():
        torch.distributed.all_reduce(t, group=group if group is not True else None)
    return t


def _copy_param(param, value):
    """param <- value without the LieTensor `__torch_function__` round trip (35 us per call, measured)."""
    with torch._C.DisableTorchFunctionSubclass():
        param.copy_(value.view(param.shape))


def _retract_se3(D, poses):
    """Exp(D) * poses for (n,6) steps and (n,7) SE3 rows.  On the GPU the two C-ABI entry points are called directly
    (the LieTensor / autograd.Function path costs ~50 us of Python per op and no graph is needed here)."""
    if D.is_cuda:
        X = _C.launch_rows("b200_se3_exp_fwd", [D.contiguous()], [7])[0]
        return _C.launch_rows("b200_SE3_mul_fwd", [X, poses.contiguous()], [7])[0]
    return (LieTensor(D, ltype=_lt.se3_type).Exp() * LieTensor(poses, ltype=SE3_type)).tensor()


def _retract_sim3(D, nodes):
    """Exp(D) * nodes for (n,7) steps and (n,8) Sim3 rows (CUDA only: the Sim3 pose-graph route runs on one GPU)."""
    X = _C.launch_rows("b200_sim3_exp_fwd", [D.contiguous()], [8])[0]
    return _C.launch_rows("b200_Sim3_mul_fwd", [X, nodes.contiguous()], [8])[0]


def _retract_so3(D, nodes):
    """Exp(D) * nodes for (n,3) steps and (n,4) SO3 rows (CUDA only: the SO3 pose-graph route runs on one GPU)."""
    X = _C.launch_rows("b200_so3_exp_fwd", [D.contiguous()], [4])[0]
    return _C.launch_rows("b200_SO3_mul_fwd", [X, nodes.contiguous()], [4])[0]


class _Problem:
    """A structured problem exposes:
         linearize()                      -> opaque state reused across the rejected trials of one step
         trial(lin, scale, dmin, dmax)    -> dict(cur=float, loss=float, predicted=float, failed=float,
                                                  cur_t=Tensor, loss_t=Tensor)    (ONE host sync)
         accept()                         -> parameters <- trial parameters
         loss()                           -> current loss (Tensor)
    """

    def _result(self, sums, order):
        """sums: small fp64 device tensor; one D2H read gives every scalar the host control flow needs."""
        vals = sums.tolist()
        r = {k: vals[i] for k, i in order.items()}
        # 0-d device views of the fp64 sums (no extra kernels); the reference's loss is a 0-d tensor too
        r["cur_t"], r["loss_t"] = sums[order["cur"]], sums[order["loss"]]
        return r


class PoseInvProblem(_Problem):
    def __init__(self, model, param, X, key, group, robust=(0, 1.0)):
        self.model, self.param, self.X, self.key, self.group = model, param, X, key, group
        self.robust = robust
        self.dtype = param.dtype
        self._trial = None
        self._same = None
        self._rows_cache = None

    def matches(self, model, input, weight=None):
        if weight is not None or model is not self.model:
            return False
        if self._same is not None and self._same.same(input):
            return True
        ok = _input_key(input) == self.key
        if ok:
            self._same = _SameInput(input)
        return ok

    def _rows(self):
        c = self._rows_cache
        if c is None or c[0] != self.param.data_ptr():          # plain (n,7) views of the parameter / input storage
            c = self._rows_cache = (self.param.data_ptr(), self.param.tensor().reshape(-1, 7), self.X.tensor().reshape(-1, 7))
        return c[1], c[2]

    def loss(self):
        P, X = self._rows()
        return _allreduce(_fused.call("lm_poseinv_loss", P, X, *self.robust), self.group)[0].to(self.dtype)

    def linearize(self):
        return None         # everything lives in registers inside the trial kernel

    def trial(self, lin, scale, dmin, dmax):
        P, X = self._rows()
        self._trial, sums = _fused.call("lm_poseinv_trial", P, X, float(scale), float(dmin), float(dmax), *self.robust)
        sums = _allreduce(sums, self.group)
        return self._result(sums, {"cur": 0, "loss": 1, "predicted": 2, "failed": 3})

    def accept(self):
        _copy_param(self.param, self._trial)

    def device_step(self, strategy):
        return _device_step(self, self.param, strategy)

    def device_trial(self, ds, scale, dmin, dmax, retry):
        if ds.comm is not None:
            return _lmstep.poseinv_trial_peer(ds, self, scale, dmin, dmax, retry)
        return _lmstep.poseinv_trial(ds, self, scale, dmin, dmax, retry)

    def peer_payload(self):
        return 0, 0, 256


class ReprojProblem(_Problem):
    def __init__(self, model, data, key, group, robust=(0, 1.0), param=None):
        self.model, self.key, self.group, self.robust = model, key, group, robust
        self.param = model.poses if param is None else param
        self.dtype = self.param.dtype
        self.pts, self.pix, self.cidx, self.seg = data
        self._trial, self._buf = None, None
        self._same = None
        self._poses_cache = None

    def matches(self, model, input, weight=None):
        if weight is not None or model is not self.model:
            return False
        if self._same is not None and self._same.same(input):
            return True
        ok = _input_key(input) == self.key
        if ok:
            self._same = _SameInput(input)
        return ok

    def _poses(self):
        c = self._poses_cache
        if c is None or c[0] != self.param.data_ptr():
            c = self._poses_cache = (self.param.data_ptr(), self.param.tensor().reshape(-1, 7))
        return c[1]

    def loss(self):
        s = _fused.call("lm_reproj_loss", self._poses(), self.pts, self.pix, self.seg, *self.robust)
        return _allreduce(s, self.group)[0].to(self.dtype)

    def _fast(self):
        return self.param.is_cuda and self.group is None

    def linearize(self):
        if self._fast():          # single rank on the GPU: caller-owned buffers, no per-kernel result clones
            poses = self._poses()
            if self._buf is None:
                C = poses.shape[0]
                self._buf = (poses.new_empty(C, 21), poses.new_empty(C, 6), torch.empty_like(poses))
            H, g, _ = self._buf
            _fused.reproj_linearize(poses, self.pts, self.pix, self.seg, *self.robust, H, g)
            return H, g, None
        H, g, s = _fused.call("lm_reproj_accum", self._poses(), self.pts, self.pix, self.seg, *self.robust)
        if self.group is not None:
            packed = torch.cat([H.reshape(-1), g.reshape(-1)])      # one packed all-reduce per LM iteration
            _allreduce(packed, self.group)
            n = H.numel()
            H, g = packed[:n].view_as(H), packed[n:].view_as(g)
        return H, g, s

    def trial(self, lin, scale, dmin, dmax):
        H, g, cur = lin
        if cur is None:
            self._trial = self._buf[2]
            sums = _fused.reproj_trial(H, g, self._poses(), self.pts, self.pix, self.seg, scale, dmin, dmax, *self.robust,
                                       self._trial)
            return self._result(sums, {"cur": 0, "loss": 4, "predicted": 8, "failed": 9})
        self._trial, _, sums = _fused.call("lm_solve6_retract", H, g, self._poses(), float(scale), float(dmin), float(dmax))
        tl = _fused.call("lm_reproj_loss", self._trial, self.pts, self.pix, self.seg, *self.robust)
        shard = torch.cat([cur, tl])                 # [current loss, trial loss] of this rank's residuals
        shard = _allreduce(shard, self.group)
        return self._result(torch.cat([shard, sums]), {"cur": 0, "loss": 1, "predicted": 2, "failed": 3})

    def accept(self):
        _copy_param(self.param, self._trial)

    def device_step(self, strategy):
        return _device_step(self, self.param, strategy)

    def device_trial(self, ds, scale, dmin, dmax, retry):
        if self._buf is None:
            poses = self._poses()
            C = poses.shape[0]
            self._buf = (poses.new_empty(C, 21), poses.new_empty(C, 6), torch.empty_like(poses))
        if ds.comm is not None:
            return _lmstep.reproj_trial_peer(ds, self, scale, dmin, dmax, retry)
        return _lmstep.reproj_trial(ds, self, scale, dmin, dmax, retry)

    def peer_payload(self):
        import torch.distributed as dist
        world = dist.get_world_size(None if self.group is True else self.group)
        return _lmstep.reproj_payload(self._poses().shape[0], world, self.param.element_size())


def _device_step(prob, param, strategy):
    """DeviceStep buffers when the device-decided route applies: CUDA parameter stored contiguously (the kernels commit
    the accepted trial straight into its storage), one rank, one of the three reference strategies."""
    if getattr(prob, '_ds', None) is not None:
        return prob._ds if _lmstep.strategy_kind(strategy) is not None else None
    if getattr(prob, '_ds_tried', False):
        return None
    prob._ds_tried = True
    if not param.is_cuda or not param.is_contiguous() or _lmstep.strategy_kind(strategy) is None:
        return None
    comm = None
    if prob.group is not None:
        # every rank reaches this point together (same model, same optimizer arguments): collective set-up of the NVLink
        # exchange; if it is not available on some rank, all ranks keep the torch.distributed route
        from .._comm import PeerComm
        part_off, pt_off, nbytes = prob.peer_payload()
        comm = PeerComm.create(prob.group, param.device, nbytes)
        if comm is None:
            return None
    prob._ds = _lmstep.DeviceStep(param.device, param.dtype)
    if comm is not None:
        prob._ds.attach_comm(comm, part_off, pt_off)
    return prob._ds


def _bmv(A, x):
    """Batched tiny mat-vec (n,k,m) @ (n,m) as one fused multiply + reduce: torch.einsum / bmm dispatches these to
    per-batch GEMV kernels that took 60-70 % of a PGO / BA step (torch.profiler, tools/prof_pgo_ba.py)."""
    return (A * x.unsqueeze(-2)).sum(-1)


def _pcg(matvec, Minv, b, tol, maxiter, check_every=4):
    """Block-Jacobi preconditioned CG on (n, 6) block vectors (the algorithm of optim/solver.py:276-340 with
    M = blockdiag(Minv)).  In-place vector updates with device-side scalars; the residual norm is read back only
    every `check_every` iterations (each read is a host sync), so up to check_every-1 extra iterations may run."""
    x = torch.zeros_like(b)
    r = b.clone()
    z = _bmv(Minv, r)
    p = z.clone()
    rz = (r * z).sum()
    stop = tol * float(b.norm())
    maxiter = maxiter if maxiter is not None else 10 * b.numel()
    it = 0
    while it < maxiter:
        if it % check_every == 0 and float(r.norm()) <= stop:
            break
        q = matvec(p)
        alpha = rz / (p * q).sum()
        x.addcmul_(p, alpha)
        r.addcmul_(q, -alpha)
        z = _bmv(Minv, r)
        rz_new = (r * z).sum()
        p.mul_(rz_new / rz).add_(z)
        rz = rz_new
        it += 1
    return x, it


_DIAG21 = [0, 6, 11, 15, 18, 20]          # positions of the 6 diagonal entries inside a packed upper triangle


def _unpack21(Hd):
    iu = torch.triu_indices(6, 6, device=Hd.device)
    A = Hd.new_zeros(Hd.shape[0], 6, 6)
    A[:, iu[0], iu[1]] = Hd
    A[:, iu[1], iu[0]] = Hd
    return A


class PGOProblem(_Problem):
    """Two-pose residuals r_e = Log(Z_e^-1 A^-1 B): block-sparse H, never assembled.

    Each trial solves (H + extra diagonal) D = -g by block-Jacobi preconditioned CG; the extra diagonal is
    clamp(diag H) * scale - diag H, i.e. the reference's clamp (optimizer.py:643/657) + cumulative damping (:664/666).

    node-ordered route (unweighted edges on one GPU; csrc/pcg2.cu, lmdrive.cu): every edge owns one slot in each
               endpoint's adjacency list, the linearisation writes its blocks there and block sums and H products are
               gathers — no atomics, bit-reproducible.
    per-edge scatter route (information matrices, or edges sharded over a process group): per-edge M_e = J^T J and
               u_e = J^T r (one kernel), diagonal blocks + gradient by atomics, a matvec that walks the edges
               (csrc/lm.cu lm_pgo_spmv_kernel).  With a group, Hd, g, every matvec and the scalars are all-reduced."""
    D = 7                       # parameter width of a node (Sim3PGOProblem: 8, SO3PGOProblem: 4)

    def __init__(self, model, edges, Z, key, group, robust, tol, maxiter, param=None, weight=None):
        self.model, self.key, self.group, self.robust = model, key, group, robust
        self.weight_key = None if weight is None else _input_key(weight)
        self.param = model.nodes if param is None else param
        self.dtype = self.param.dtype
        self.ei = edges[..., 0].to(torch.int32).contiguous()
        self.ej = edges[..., 1].to(torch.int32).contiguous()
        self.Z = None if Z is None else Z.tensor().to(self.dtype).reshape(-1, self.D).contiguous()
        # information matrices (examples/module/pgo/pgo.py:75 `weight=infos`): (E,6,6) or one (6,6) for all edges
        self.W = None if weight is None else weight.to(self.dtype).reshape(-1, 36).contiguous()
        self.kind = "pgo"
        # node adjacency of the node-ordered route: each edge's slot in the lists of its two endpoints
        E = self.ei.shape[0]
        keys = torch.cat([self.ei, self.ej]).long()
        order = torch.sort(keys, stable=True)[1]
        self.nother = torch.cat([self.ej, self.ei])[order].contiguous()
        N = self.param.tensor().reshape(-1, self.D).shape[0]
        self.nptr = torch.zeros(N + 1, dtype=torch.int32, device=keys.device)
        self.nptr[1:] = torch.cumsum(torch.bincount(keys, minlength=N), 0).to(torch.int32)
        pos = torch.empty(2 * E, dtype=torch.int32, device=keys.device)
        pos[order] = torch.arange(2 * E, dtype=torch.int32, device=keys.device)
        self.epos_i, self.epos_j = pos[:E].contiguous(), pos[E:].contiguous()
        self.tol, self.maxiter = tol, maxiter
        self._trial = None
        self.cg_iters = 0

    def matches(self, model, input, weight=None):
        return (model is self.model and _input_key(input) == self.key
                and self.weight_key == (None if weight is None else _input_key(weight)))

    def _nodes(self):
        return self.param.tensor().reshape(-1, self.D)

    # the two family-specific pieces (overridden by Reproj2Problem): per-edge blocks and the loss at given nodes
    def _loss_at(self, nodes):
        return _fused.call("lm_pgo_loss", nodes, self.Z, self.ei, self.ej, *self.robust)

    def _blocks(self, nodes):
        """-> M (E,21), u (E,6), cost (1,), unweighted (M0, u0) or None"""
        if self.W is None:
            M, u, cur = _fused.call("lm_pgo_linearize", nodes, self.Z, self.ei, self.ej, *self.robust)
            return M, u, cur, None
        M, u, M0, u0, cur = _fused.call("lm_pgo_linearize_w", nodes, self.Z, self.ei, self.ej, self.W, *self.robust)
        return M, u, cur, (M0, u0)

    def loss(self):
        return _allreduce(self._loss_at(self._nodes()), self.group)[0].to(self.dtype)

    def linearize(self):
        nodes = self._nodes()
        if nodes.is_cuda and self.group is None and self.W is None:
            Mn, Hd, g, cur = _fused.pgo_linearize_nodes(self.kind, self, nodes, *self.robust)
            return (Mn,), Hd, g, cur, None
        M, u, cur, unw = self._blocks(nodes)
        comm = self._peer(27 * nodes.shape[0]) if (M.is_cuda and self.group is not None) else None
        if comm is not None:      # multi-GPU device route: [Hd | g] of this rank's edges, one device all-reduce
            n = nodes.shape[0]
            packed = torch.zeros(n * 27, dtype=M.dtype, device=M.device)
            Hd, g = packed[:n * 21].view(n, 21), packed[n * 21:].view(n, 6)
            _fused._launch("b200_lm_pgo_scatter", M, [M.data_ptr(), u.data_ptr(), self.ei.data_ptr(), self.ej.data_ptr(),
                                                      Hd.data_ptr(), g.data_ptr()], M.shape[0])
            comm.sum_(packed)
            return M, Hd, g, cur, (unw if unw is not None else (M, u))      # predicted from the per-edge blocks
        Hd, g = _fused.call("lm_pgo_scatter", M, u, self.ei, self.ej, nodes.shape[0])
        if self.group is not None:
            packed = torch.cat([Hd.reshape(-1), g.reshape(-1)])
            _allreduce(packed, self.group)
            n = Hd.numel()
            Hd, g = packed[:n].view_as(Hd), packed[n:].view_as(g)
        return M, Hd, g, cur, unw

    def _matvec(self, M, extra, x):
        y = _fused.call("lm_pgo_spmv", M, self.ei, self.ej, x, torch.zeros_like(x))
        return _allreduce(y, self.group) + extra * x

    def trial(self, lin, scale, dmin, dmax):
        M, Hd, g, cur, unw = lin
        comm = getattr(self, '_comm', None)
        if isinstance(M, tuple):                                          # node-ordered blocks: csrc/pcg2.cu
            D, self.cg_iters, predicted = _fused.pgo_solve_nodes(M[0], self.nother, self.nptr, Hd, g, scale, dmin, dmax,
                                                                 self.tol, self.maxiter,
                                                                 hint=self.cg_iters + 1 if self.cg_iters else 0)
            return self._finish_trial(D, predicted, cur)
        if M.is_cuda and (self.group is None or comm is not None):       # device-resident PCG on per-edge blocks
            D, self.cg_iters, predicted = _fused.pgo_solve(M, self.ei, self.ej, Hd, g, scale, dmin, dmax, self.tol,
                                                           self.maxiter, hint=self.cg_iters + 1 if self.cg_iters else 0,
                                                           unweighted=unw, comm=comm)
            if comm is not None:
                predicted = _allreduce(predicted, self.group)
            return self._finish_trial(D, predicted, cur)
        d = Hd[:, _DIAG21]
        extra = d.clamp(dmin, dmax) * scale - d                       # added to the diagonal of H
        blocks = _unpack21(Hd) + torch.diag_embed(extra)
        Minv = torch.linalg.inv(blocks)                               # block-Jacobi preconditioner
        x, it = _pcg(lambda v: self._matvec(M, extra, v), Minv, -g, self.tol, self.maxiter)
        self.cg_iters = it
        D = x
        if unw is None:
            Hx = _fused.call("lm_pgo_spmv", M, self.ei, self.ej, D, torch.zeros_like(D))
            Hx = _allreduce(Hx, self.group)
            predicted = ((D * Hx).sum() + 2 * (D * g).sum()).to(torch.float64).reshape(1)
        else:     # (J D)^T (2 R + J D) without the weights (strategy.py:143): per-edge sum over this rank's edges
            d = D[self.ej.long()] - D[self.ei.long()]
            predicted = ((d * _bmv(_unpack21(unw[0]), d)).sum() + 2 * (d * unw[1]).sum()).to(torch.float64).reshape(1)
            predicted = _allreduce(predicted, self.group)
        return self._finish_trial(D, predicted, cur)

    def _retract(self, D, nodes):
        return _retract_se3(D, nodes)

    def _finish_trial(self, D, predicted, cur):
        self._trial = self._retract(D, self._nodes())
        tl = self._loss_at(self._trial)
        shard = _allreduce(torch.cat([cur, tl]), self.group)
        return self._result(torch.cat([shard, predicted, predicted.new_zeros(1)]),
                            {"cur": 0, "loss": 1, "predicted": 2, "failed": 3})

    def accept(self):
        _copy_param(self.param, self._trial)

    def _peer(self, max_elems):
        return _peer_allreduce(self, self.param, max_elems)

    # one C call per trial (csrc/lmdrive.cu): single GPU, node-ordered blocks, no information matrices
    def device_step(self, strategy):
        if getattr(self, '_pds', None) is not None:
            return self._pds if _lmstep.strategy_kind(strategy) is not None else None
        if getattr(self, '_pds_tried', False):
            return None
        self._pds_tried = True
        nodes = self._nodes()
        if (not nodes.is_cuda or self.group is not None or self.W is not None
                or _lmstep.strategy_kind(strategy) is None or not self.param.is_contiguous()
                or nodes.get_device() != torch.cuda.current_device()):
            return None
        self._pds = _lmstep.PgoDeviceStep(self, nodes)
        return self._pds

    def device_trial(self, ds, scale, dmin, dmax, retry):
        return ds.trial(self, self._nodes(), scale, dmin, dmax, retry)


class Reproj2Problem(PGOProblem):
    """Two-pose reprojection r = proj(T_b^-1 T_a p) - z (module.TwoPoseReproj; BASELINE.json configs[4] as stated).
    d r / d xi_b = -d r / d xi_a, so all rows of one ordered pair (a, b) add into one 6x6 block and the pairs are the edges
    of the pose-graph machinery above: rows are sorted by pair once, csrc/lm.cu lm_reproj2_accum gives (M, u) per pair in
    one warp-per-pair pass over 20 B per row, everything after that (block diagonal, device PCG, retraction, multi-GPU
    reduction) is inherited.  Sign convention of PGOProblem: edge (ei, ej) has J_ei = -J, J_ej = +J  =>  ei = b, ej = a."""

    def __init__(self, model, points, pixels, ia, ib, intr, key, group, robust, tol, maxiter, param=None):
        param = model.poses if param is None else param
        N = param.tensor().reshape(-1, 7).shape[0]
        ia, ib = ia.reshape(-1).long(), ib.reshape(-1).long()
        order = torch.sort(ia * N + ib, stable=True)[1]
        pair_key = (ia * N + ib)[order]
        uniq, counts = torch.unique_consecutive(pair_key, return_counts=True)
        pa, pb = (uniq // N), (uniq % N)
        super().__init__(model, torch.stack([pb, pa], 1), None, key, group, robust, tol, maxiter, param=param)
        self.pa, self.pb = pa.to(torch.int32).contiguous(), pb.to(torch.int32).contiguous()
        self.pseg = torch.zeros(uniq.numel() + 1, dtype=torch.int32, device=ia.device)
        self.pseg[1:] = torch.cumsum(counts, 0).to(torch.int32)
        self.pts = points.reshape(-1, 3)[order].to(self.dtype).contiguous()
        self.pix = pixels.reshape(-1, 2)[order].to(self.dtype).contiguous()
        self.intr = tuple(float(v) for v in intr)
        self.kind = "reproj2"

    def _loss_at(self, nodes):
        return _fused.call("lm_reproj2_loss", nodes, self.pts, self.pix, self.pseg, self.pa, self.pb, self.intr, *self.robust)

    def _blocks(self, nodes):
        M, u, cur = _fused.call("lm_reproj2_accum", nodes, self.pts, self.pix, self.pseg, self.pa, self.pb, self.intr,
                                *self.robust)
        return M, u, cur, None


class Sim3PGOProblem(PGOProblem):
    """Sim3 pose graph r_e = Log(Z_e^-1 A^-1 B) on Sim3 nodes (examples/module/pgo `PoseGraph` with pp.Sim3 nodes, as in
    monocular loop closure, where scale drifts).  A node has 7 unknowns [tau phi sigma]; J = sim3_Jl_inv(r) Adj(Z^-1 A^-1)
    with the reference's truncated series (csrc/sim3pgo_math.cuh).  The blocks are written in node order and solved by the
    PCG of csrc/pcg2.cu at block width 7; the update is Exp(D) P.  One CUDA device, no process group, no information
    matrices (those graphs keep the generic route)."""
    D = 8

    def __init__(self, model, edges, Z, key, robust, tol, maxiter, param=None):
        super().__init__(model, edges, Z, key, None, robust, tol, maxiter, param=param)
        self.kind = "sim3"

    def _loss_at(self, nodes):
        return _fused.sim3pgo_loss(nodes, self.Z, self.ei, self.ej, *self.robust)

    def linearize(self):
        Mn, Hd, g, cur = _fused.pgo_linearize_nodes(self.kind, self, self._nodes(), *self.robust)
        return (Mn,), Hd, g, cur, None

    def _retract(self, D, nodes):
        return _retract_sim3(D, nodes)


class SO3PGOProblem(PGOProblem):
    """SO3 pose graph r_e = Log(Z_e^-1 A^-1 B) on SO3 nodes (examples/module/pgo `PoseGraph` with pp.SO3 nodes): rotation
    averaging, the first stage of global structure from motion.  A node has 3 unknowns; J = so3_Jl_inv(r) R(Z^-1 A^-1)
    (csrc/so3pgo_math.cuh).  The blocks are written in node order and solved by the PCG of csrc/pcg2.cu at block width 3;
    the update is Exp(D) P.  One CUDA device, no process group, no information matrices (those graphs keep the generic
    route)."""
    D = 4

    def __init__(self, model, edges, Z, key, robust, tol, maxiter, param=None):
        super().__init__(model, edges, Z, key, None, robust, tol, maxiter, param=param)
        self.kind = "so3"

    def _loss_at(self, nodes):
        return _fused.so3pgo_loss(nodes, self.Z, self.ei, self.ej, *self.robust)

    def linearize(self):
        Mn, Hd, g, cur = _fused.pgo_linearize_nodes(self.kind, self, self._nodes(), *self.robust)
        return (Mn,), Hd, g, cur, None

    def _retract(self, D, nodes):
        return _retract_so3(D, nodes)


def _peer_allreduce(prob, param, max_elems):
    """NVLink exchange for the device all-reduces of a sharded block-sparse problem (collective set-up on first use; None
    keeps the torch.distributed route)."""
    if not getattr(prob, '_comm_tried', False):
        prob._comm_tried = True
        from .._comm import PeerComm
        prob._comm = PeerComm.for_allreduce(prob.group, param.device, int(max_elems), param.element_size())
    return prob._comm


def _unpack6(Hp):
    """(P, 6) packed upper triangles of 3x3 blocks -> (P, 3, 3)."""
    iu = torch.triu_indices(3, 3, device=Hp.device)
    A = Hp.new_zeros(Hp.shape[0], 3, 3)
    A[:, iu[0], iu[1]] = Hp
    A[:, iu[1], iu[0]] = Hp
    return A


def _group_by_camera(prob, pix, cidx, pidx, C, P):
    """Observation layout of the deterministic bundle-adjustment routes (csrc/ba.cu, csrc/bal.cu), set on `prob`."""
    # observations are regrouped by camera once (the LM sums do not depend on their order): the camera-side
    # scatter-adds of the kernels then collapse to one atomic per warp and value (csrc/lm_common.cuh seg_atomic_add)
    order = torch.sort(cidx.reshape(-1), stable=True)[1]
    pix, cidx, pidx = pix.reshape(-1, 2)[order], cidx.reshape(-1)[order], pidx.reshape(-1)[order]
    prob.pix = pix.to(prob.dtype).contiguous()
    prob.cidx, prob.pidx = cidx.to(torch.int32).contiguous(), pidx.to(torch.int32).contiguous()
    prob.cl, prob.pl = cidx.long(), pidx.long()
    # observation ids grouped by point (CSR): W^T x of the device PCG gathers along it instead of scatter-adding
    prob.padj = torch.sort(prob.pl, stable=True)[1].contiguous()
    prob.cidx_p = prob.cidx[prob.padj].contiguous()
    prob.ppos = torch.empty_like(prob.padj, dtype=torch.int32)          # inverse permutation: position in point order
    prob.ppos[prob.padj] = torch.arange(prob.padj.numel(), dtype=torch.int32, device=prob.padj.device)
    prob.pptr = torch.zeros(P + 1, dtype=torch.int32, device=prob.pl.device)
    prob.pptr[1:] = torch.cumsum(torch.bincount(prob.pl, minlength=P), 0).to(torch.int32)
    # geometry of the deterministic device route (csrc/ba.cu): rows per camera, work items per camera (so that a few
    # cameras with very many rows still fill the machine) and threads per item, point-ordered pixels
    m = prob.cidx.numel()
    prob.cseg = torch.zeros(C + 1, dtype=torch.int32, device=prob.pl.device)
    prob.cseg[1:] = torch.cumsum(torch.bincount(prob.cl, minlength=C), 0).to(torch.int32)
    tpi = 128 if m >= 192 * C else 32
    sms = _sms(prob.pl.device) if prob.pl.is_cuda else 132     # the geometry only steers the device kernels
    want = sms * 8 * (128 // tpi)                      # items that fill the SMs
    split = max(1, min(want // max(C, 1), (m // max(C, 1)) // (8 * tpi))) if C < want else 1
    prob.geom = (prob.cseg, int(split), int(tpi), prob.ppos, prob.cidx_p, prob.pptr, prob.pix[prob.padj].contiguous())


class BAProblem(_Problem):
    """Bundle adjustment with poses (C,7) and points (P,3) as parameters, in the reference's parameter order.

    The normal equations [[Hcc, W], [W^T, Hpp]] [dc; dp] = -[gc; gp] (diagonal clamped + damped like the dense
    branch, optimizer.py:657/666) are solved by eliminating the 3x3 point blocks:
        (Hcc - W Hpp^-1 W^T) dc = -gc + W Hpp^-1 gp,     dp = Hpp^-1 (-gp - W^T dc)
    with a block-Jacobi preconditioned CG whose W / W^T products walk the observations (csrc/lm.cu lm_ba_wv / wtx).
    Observations may be sharded over a process group (blocks, gradients and every product all-reduced)."""

    def __init__(self, model, pix, cidx, pidx, key, group, robust, tol, maxiter, params=None):
        self.model, self.key, self.group, self.robust = model, key, group, robust
        self.poses, self.points = (model.poses, model.points_3d) if params is None else params
        self.dtype = self.poses.dtype
        C, P = self.poses.tensor().reshape(-1, 7).shape[0], self.points.reshape(-1, 3).shape[0]
        _group_by_camera(self, pix, cidx, pidx, C, P)
        self.tol, self.maxiter = tol, maxiter
        self._trial = None
        self.cg_iters = 0

    def matches(self, model, input, weight=None):
        return weight is None and model is self.model and _input_key(input) == self.key

    def _params(self):
        return self.poses.tensor().reshape(-1, 7), self.points.reshape(-1, 3)

    def loss(self):
        T, p = self._params()
        s = _fused.call("lm_ba_loss", T, p, self.pix, self.cidx, self.pidx, *self.robust)
        return _allreduce(s, self.group)[0].to(self.dtype)

    def linearize(self):
        T, p = self._params()
        comm = None
        if T.is_cuda and self.group is not None:
            comm = _peer_allreduce(self, self.poses, max(27 * T.shape[0] + 9 * p.shape[0], 3 * p.shape[0]))
        if T.is_cuda and (self.group is None or comm is not None):   # device PCG route: 16 B per observation, no atomics
            Y4s, rs, Hcc, Hpp, gc, gp, cur = _fused.ba_linearize_det(T, p, self.pix, self.pidx, self.geom, *self.robust)
            if comm is not None:          # block sums of this rank's observations -> one device all-reduce
                packed = torch.cat([t.reshape(-1) for t in (Hcc, Hpp, gc, gp)])
                comm.sum_(packed)
                outs, o = [], 0
                for t in (Hcc, Hpp, gc, gp):
                    outs.append(packed[o:o + t.numel()].view_as(t)); o += t.numel()
                Hcc, Hpp, gc, gp = outs
            return Y4s, T, rs, Hcc, Hpp, gc, gp, cur
        Jc, Jp, rs, Hcc, Hpp, gc, gp, cur = _fused.call("lm_ba_linearize", T, p, self.pix, self.cidx, self.pidx, *self.robust)
        if self.group is not None:
            packed = torch.cat([t.reshape(-1) for t in (Hcc, Hpp, gc, gp)])
            _allreduce(packed, self.group)
            outs, o = [], 0
            for t in (Hcc, Hpp, gc, gp):
                outs.append(packed[o:o + t.numel()].view_as(t)); o += t.numel()
            Hcc, Hpp, gc, gp = outs
        return Jc, Jp, rs, Hcc, Hpp, gc, gp, cur

    def trial(self, lin, scale, dmin, dmax):
        Jc, Jp, rs, Hcc, Hpp, gc, gp, cur = lin
        C, P = Hcc.shape[0], Hpp.shape[0]
        if isinstance(Jc, tuple):                     # device-resident Schur PCG; (Jc, Jp) are ((Y4, Y4p), poses) here
            xc, xp, self.cg_iters, pred = _fused.ba_solve(Jc, Jp, rs, self.cidx, self.pidx, self.geom, Hcc, Hpp,
                                                          gc, gp, scale, dmin,
                                                          dmax, self.tol, self.maxiter, hint=self.cg_iters + 1 if self.cg_iters else 0,
                                                          comm=getattr(self, '_comm', None))
            return self._finish_trial(xc, xp, pred, cur)
        dc, dp = Hcc[:, _DIAG21], Hpp[:, [0, 3, 5]]
        Hc = _unpack21(Hcc) + torch.diag_embed(dc.clamp(dmin, dmax) * scale - dc)
        Hp_inv = torch.linalg.inv(_unpack6(Hpp) + torch.diag_embed(dp.clamp(dmin, dmax) * scale - dp))

        def WTx(x):
            return _allreduce(_fused.call("lm_ba_wtx", Jc, Jp, self.cidx, self.pidx, x, P), self.group)

        def Wv(v):
            return _allreduce(_fused.call("lm_ba_wv", Jc, Jp, self.cidx, self.pidx, v, C), self.group)

        def pinv(t):
            return _bmv(Hp_inv, t)

        def S(x):                                     # reduced camera system
            return _bmv(Hc, x) - Wv(pinv(WTx(x)))

        # block-Jacobi preconditioner on the Schur diagonal: Hc - sum_k (Jc^T Jp) Hp^-1 (Jp^T Jc)
        Jc3, Jp3 = Jc.view(-1, 2, 6), Jp.view(-1, 2, 3)
        Wk = Jc3[:, 0, :, None] * Jp3[:, 0, None, :] + Jc3[:, 1, :, None] * Jp3[:, 1, None, :]          # (m,6,3) = Jc^T Jp
        WH = (Wk.unsqueeze(-1) * Hp_inv[self.pl].unsqueeze(1)).sum(-2)                                  # (m,6,3) = Wk Hp^-1
        Tk = (WH.unsqueeze(2) * Wk.unsqueeze(1)).sum(-1)                                                # (m,6,6)
        Sd = Hc.clone().index_add_(0, self.cl, -Tk)
        if self.group is not None:       # every rank added its local -Tk to the already reduced Hc
            Sd = Hc + _allreduce(Sd - Hc, self.group)
        Minv = torch.linalg.inv(Sd)
        x, it = _pcg(S, Minv, -gc + Wv(pinv(gp)), self.tol, self.maxiter)
        self.cg_iters = it
        xc = x
        xp = pinv(-gp - WTx(xc))
        # predicted = (J D)^T (2 R + J D), per observation (corrected J and R)
        Jd = _bmv(Jc3, xc[self.cl]) + _bmv(Jp3, xp[self.pl])
        pred = ((Jd * Jd).sum() + 2 * (rs * Jd).sum()).to(torch.float64).reshape(1)
        return self._finish_trial(xc, xp, pred, cur)

    def _finish_trial(self, xc, xp, pred, cur):
        T, pts = self._params()
        Tn = _retract_se3(xc, T)
        pn = pts + xp
        self._trial = (Tn, pn)
        tl = _fused.call("lm_ba_loss", Tn, pn, self.pix, self.cidx, self.pidx, *self.robust)
        shard = _allreduce(torch.cat([cur, tl, pred]), self.group)
        return self._result(torch.cat([shard, shard.new_zeros(1)]), {"cur": 0, "loss": 1, "predicted": 2, "failed": 3})

    def accept(self):
        _copy_param(self.poses, self._trial[0])
        _copy_param(self.points, self._trial[1])

    # one C call per trial (csrc/lmdrive.cu b200_lm_ba_step): single GPU
    def device_step(self, strategy):
        if getattr(self, '_bds', None) is not None:
            return self._bds if _lmstep.strategy_kind(strategy) is not None else None
        if getattr(self, '_bds_tried', False):
            return None
        self._bds_tried = True
        T, p = self._params()
        if (not T.is_cuda or self.group is not None or _lmstep.strategy_kind(strategy) is None
                or not self.poses.is_contiguous() or not self.points.is_contiguous() or T.dtype != p.dtype
                or T.get_device() != torch.cuda.current_device()):
            return None
        self._bds = _lmstep.BaDeviceStep(self, T, p)
        return self._bds

    def device_trial(self, ds, scale, dmin, dmax, retry):
        T, p = self._params()
        return ds.trial(self, T, p, scale, dmin, dmax, retry)


class BALProblem(_Problem):
    """BAL bundle adjustment (module.BALBundleAdjustment, the reference's examples/module/ba `Reproj(K, C, P)`): per-camera
    intrinsics (C,3) = (f, k1, k2), poses (C,7) and points (P,3).  The unknowns of a camera are [xi | f, k1, k2] (9), of
    a point dp (3); J^T J over all of them is clamped and damped like the dense branch (optimizer.py:657/666) and solved by
    eliminating the 3x3 point blocks, as BAProblem does, with a device PCG over 9-wide camera blocks (csrc/bal.cu, no
    atomics).  The update is Exp(xi) T for the poses and addition for intrinsics and points.  One CUDA device, no
    process group, no residual weights."""

    def __init__(self, model, pix, cidx, pidx, key, robust, tol, maxiter, params):
        self.model, self.key, self.group, self.robust = model, key, None, robust
        self.intr, self.poses, self.points = params
        self.dtype = self.poses.dtype
        _group_by_camera(self, pix, cidx, pidx, self.poses.shape[0], self.points.shape[0])
        self.tol, self.maxiter = tol, maxiter
        self._trial = None
        self.cg_iters = 0

    def matches(self, model, input, weight=None):
        return weight is None and model is self.model and _input_key(input) == self.key

    def _params(self):
        return self.intr.reshape(-1, 3), self.poses.tensor().reshape(-1, 7), self.points.reshape(-1, 3)

    def loss(self):
        K, T, p = self._params()
        return _fused.bal_loss(K, T, p, self.pix, self.cidx, self.pidx, *self.robust)[0].to(self.dtype)

    def linearize(self):
        K, T, p = self._params()
        return _fused.bal_linearize(K, T, p, self.pix, self.pidx, self.geom, *self.robust)

    def trial(self, lin, scale, dmin, dmax):
        Y4s, rs, Hcc, Hpp, gc, gp, cur = lin
        K, T, p = self._params()
        xc, xp, self.cg_iters, pred = _fused.bal_solve(Y4s, K, T, rs, self.cidx, self.pidx, self.geom, Hcc, Hpp, gc, gp,
                                                       scale, dmin, dmax, self.tol, self.maxiter,
                                                       hint=self.cg_iters + 1 if self.cg_iters else 0)
        self._trial = _fused.bal_retract(K, T, p, xc, xp)
        tl = _fused.bal_loss(*self._trial, self.pix, self.cidx, self.pidx, *self.robust)
        sums = torch.cat([cur, tl, pred, pred.new_zeros(1)])
        return self._result(sums, {"cur": 0, "loss": 1, "predicted": 2, "failed": 3})

    def accept(self):
        _copy_param(self.intr, self._trial[0])
        _copy_param(self.poses, self._trial[1])
        _copy_param(self.points, self._trial[2])

    def device_step(self, strategy):
        return None                 # every trial is driven from the host (LevenbergMarquardt._step_structured)


def _input_key(input):
    items = input if isinstance(input, (tuple, list)) else (input,)
    return tuple((t.data_ptr(), tuple(t.shape), t.dtype, t._version) if torch.is_tensor(t) else id(t) for t in items)


class _SameInput:
    """`matches` asks every step whether (model, input) is still the problem that was prepared (sorted copies, CSR
    offsets).  The usual caller passes the very same tensors again: identity of the objects plus their in-place version
    counters answers that in ~1 us; anything else falls back to the full key."""
    __slots__ = ("items", "versions")

    def __init__(self, input):
        self.items = tuple(input) if isinstance(input, (tuple, list)) else (input,)
        self.versions = tuple(t._version if torch.is_tensor(t) else 0 for t in self.items)

    def same(self, input):
        items = input if isinstance(input, (tuple, list)) else (input,)
        if len(items) != len(self.items):
            return False
        for a, b, v in zip(items, self.items, self.versions):
            if a is not b or (torch.is_tensor(a) and a._version != v):
                return False
        return True


def _is_se3_param(p):
    return isinstance(p, Parameter) and getattr(p, 'ltype', None) is SE3_type and p.requires_grad and p.is_cuda is not None


def _prepare_reproj(param, points, pixels, cidx):
    """Sort observations by camera and build per-camera row offsets (same as PoseReproj.prepare)."""
    C = param.shape[0]
    order = torch.argsort(cidx, stable=True)
    c_sorted = cidx[order]
    seg = torch.zeros(C + 1, dtype=torch.int32, device=cidx.device)
    seg[1:] = torch.cumsum(torch.bincount(c_sorted, minlength=C), 0).to(torch.int32)
    dt = param.dtype
    return points[order].to(dt).contiguous(), pixels[order].to(dt).contiguous(), c_sorted.to(torch.int32).contiguous(), seg


def _in_range(idx, n):
    """All indices in [0, n) — the fused kernels gather without bounds checks (one host read, at recognition only)."""
    return idx.numel() == 0 or bool(((idx >= 0) & (idx < n)).all())


def _is_index(t, n=None):
    return torch.is_tensor(t) and t.dtype in (torch.int64, torch.int32) and t.dim() == 1 and (n is None or t.shape[0] == n)


def _recognize_by_signature(model, input, params, group, robust, solver, sparse, weight=None):
    """User-written modules (e.g. README.md:163-198 `Reproj`, examples/module/pgo `PoseGraph`) reach a fused family
    when (i) their parameters and inputs have the family's types and shapes and (ii) the output of ONE eager forward
    pass has the family's shape and the same sum of squares as the family's residual kernel on the same data
    (relative 1e-4).  Anything else falls through to the generic dense route."""
    from .solver import CG
    if len(params) == 3:
        return _recognize_bal(model, input, params, group, robust, solver, sparse, weight)
    if not isinstance(input, (tuple, list)) or len(params) not in (1, 2) or not _is_se3_param(params[0]):
        return None
    if params[0].dim() != 2 or params[0].dtype not in (torch.float32, torch.float64):
        return None
    iterative = isinstance(solver, CG) or sparse
    tol = solver.tol if isinstance(solver, CG) else 1e-8
    maxiter = solver.maxiter if isinstance(solver, CG) else None
    key, cand, M, d = _input_key(input), None, None, None
    if len(params) == 2 and iterative and len(input) == 3:                           # bundle adjustment
        pts, (obs, ci, pi_) = params[1], input
        if (torch.is_tensor(pts) and not isinstance(pts, LieTensor) and pts.dim() == 2 and pts.shape[1] == 3
                and torch.is_tensor(obs) and obs.dim() == 2 and obs.shape[1] == 2 and _is_index(ci, obs.shape[0])
                and _is_index(pi_, obs.shape[0]) and _in_range(ci, params[0].shape[0]) and _in_range(pi_, pts.shape[0])):
            cand = BAProblem(model, obs, ci, pi_, key, group, (0, 1.0), tol, maxiter, params=(params[0], pts))
            M, d = obs.shape[0], 2
    elif len(params) == 1 and len(input) == 2 and iterative:                         # pose graph
        edges, Z = input
        if (torch.is_tensor(edges) and edges.dtype in (torch.int64, torch.int32) and edges.dim() == 2 and edges.shape[1] == 2
                and isinstance(Z, LieTensor) and Z.ltype is SE3_type and Z.shape == (edges.shape[0], 7)
                and _in_range(edges, params[0].shape[0])):
            cand = PGOProblem(model, edges, Z, key, group, (0, 1.0), tol, maxiter, param=params[0], weight=weight)
            M, d = edges.shape[0], 6
    elif len(params) == 1 and len(input) == 3 and not isinstance(solver, CG):        # single-pose reprojection
        points, pixels, ci = input
        if (torch.is_tensor(points) and points.dim() == 2 and points.shape[1] == 3 and torch.is_tensor(pixels)
                and pixels.shape == (points.shape[0], 2) and _is_index(ci, points.shape[0])
                and _in_range(ci, params[0].shape[0])):
            cand = ReprojProblem(model, _prepare_reproj(params[0], points, pixels, ci), key, group, (0, 1.0), param=params[0])
            M, d = points.shape[0], 2
    if cand is None or (weight is not None and not isinstance(cand, PGOProblem)):
        return None
    if not _same_residuals(model, input, params, (M, d), group):
        return None
    cand.robust = robust
    return cand


def _bal_residuals(input, K, T, P):
    """Row-wise residuals of the BAL model (examples/module/ba `Reproj.project` - observations) with LieTensor ops."""
    obs, ci, pi_ = input
    ci = ci.long()
    y = LieTensor(T.detach(), ltype=SE3_type)[ci].Act(P.detach()[pi_.long()])
    n = -y[..., :2] / y[..., 2:]
    rho = n.square().sum(-1, keepdim=True)
    k = K.detach()[ci]
    return k[..., :1] * (1 + k[..., 1:2] * rho + k[..., 2:3] * rho.square()) * n - obs


def _bal_params_ok(K, T, P):
    """(C,3) intrinsics, SE3 (C,7) poses and (P,3) points of one floating dtype on one CUDA device."""
    return (_is_se3_param(T) and T.dim() == 2 and T.is_cuda and T.dtype in (torch.float32, torch.float64)
            and all(torch.is_tensor(t) and not isinstance(t, LieTensor) and t.dim() == 2 and t.shape[1] == 3
                    and t.dtype == T.dtype and t.device == T.device for t in (K, P))
            and K.shape[0] == T.shape[0])


def _recognize_lie_pgo(model, input, params, group, robust, solver, sparse, weight):
    """A pose graph on Sim3 or SO3 nodes takes its node-ordered route (Sim3PGOProblem / SO3PGOProblem, chosen by the
    parameter's ltype) when an iterative solve was asked for (solver=PCG()/CG() or sparse=True), the one trainable
    parameter is an (N,D) Parameter of that group on a CUDA device, the input is (edges (E,2) in range, Z (E,D) of the same
    group) of the parameter's dtype and device, there are no information matrices and no process group, and the model is
    the built-in PoseGraph or its output equals the pose-graph residual row by row (_same_residuals)."""
    from .solver import CG
    from ..module.pgo import PoseGraph
    P = params[0]
    ltype = P.ltype
    if not (isinstance(solver, CG) or sparse) or weight is not None or group is not None:
        return None
    if not (isinstance(P, Parameter) and P.is_cuda and P.dim() == 2 and P.dtype in (torch.float32, torch.float64)):
        return None
    if not isinstance(input, (tuple, list)) or len(input) != 2:
        return None
    edges, Z = input
    if not (torch.is_tensor(edges) and edges.dtype in (torch.int64, torch.int32) and edges.dim() == 2 and edges.shape[1] == 2
            and edges.device == P.device and isinstance(Z, LieTensor) and Z.ltype is ltype
            and Z.shape == (edges.shape[0], ltype.D) and Z.dtype == P.dtype and Z.device == P.device):
        return None
    tol = solver.tol if isinstance(solver, CG) else 1e-8
    maxiter = solver.maxiter if isinstance(solver, CG) else None
    if _is_builtin(model, PoseGraph):
        if P is not model.nodes:
            return None
        if not _in_range(edges, P.shape[0]):
            raise IndexError("PoseGraph: edge index out of range")
    elif not (_in_range(edges, P.shape[0]) and _same_residuals(model, input, params, (edges.shape[0], ltype.K), group)):
        return None
    return _LIE_PGO[ltype](model, edges, Z, _input_key(input), robust, tol, maxiter, param=P)


_LIE_PGO = {Sim3_type: Sim3PGOProblem, SO3_type: SO3PGOProblem}


def recognize_so3_graph(model, input, params, group=None, robust=(0, 1.0), solver=None, sparse=False, weight=None):
    """SO3PGOProblem for an SO3 pose graph (rotation averaging) under the conditions of _recognize_lie_pgo, else None.
    `recognize` keeps returning None for SO3 graphs, as it always has: the LM asks for this family only where it would
    otherwise build per-residual blocks (an iterative solve, no weight), which is where the SO3 route replaces them."""
    params = [p for p in params if p.requires_grad]
    if not (len(params) == 1 and getattr(params[0], 'ltype', None) is SO3_type):
        return None
    return _recognize_lie_pgo(model, input, params, group, robust, solver, sparse, weight)


def _recognize_bal(model, input, params, group, robust, solver, sparse, weight):
    """A user module with three trainable parameters takes the BAL route when they are a plain (C,3), an SE3 (C,7) and a
    plain (P,3), the input is (pixels (M,2), camera indices, point indices) in range, and its output equals the BAL
    residual row by row (_same_residuals).  With P == C the shapes cannot tell intrinsics from points: both assignments
    are tried."""
    from .solver import CG
    if not (isinstance(solver, CG) or sparse) or weight is not None or group is not None:
        return None
    if not isinstance(input, (tuple, list)) or len(input) != 3:
        return None
    obs, ci, pi_ = input
    if not (torch.is_tensor(obs) and obs.dim() == 2 and obs.shape[1] == 2 and _is_index(ci, obs.shape[0])
            and _is_index(pi_, obs.shape[0])):
        return None
    se3 = [p for p in params if _is_se3_param(p)]
    if len(se3) != 1:
        return None
    T = se3[0]
    K0, K1 = [p for p in params if p is not T]
    for K, P in ((K0, K1), (K1, K0)):
        if not (_bal_params_ok(K, T, P) and _in_range(ci, T.shape[0]) and _in_range(pi_, P.shape[0])):
            continue
        if _same_residuals(model, input, params, (obs.shape[0], 2), group, roles=(K, T, P)):
            tol = solver.tol if isinstance(solver, CG) else 1e-8
            maxiter = solver.maxiter if isinstance(solver, CG) else None
            return BALProblem(model, obs, ci, pi_, _input_key(input), robust, tol, maxiter, (K, T, P))
    return None


def _family_residuals(input, params):
    """Row-wise residuals of the family the shapes point at, from the *original* (unsorted) inputs with ordinary
    LieTensor ops — an independent restatement used only to verify a user module at recognition time."""
    T = LieTensor(params[0].detach(), ltype=params[0].ltype)      # SE3, or Sim3 / SO3 for those pose graphs
    if len(params) == 2:                                          # bundle adjustment
        obs, ci, pi_ = input
        y = T[ci.long()].Act(params[1].detach()[pi_.long()])
        return -y[..., :2] / y[..., 2:] - obs
    if len(input) == 2:                                           # pose graph
        edges, Z = input
        return (Z.Inv() @ T[edges[:, 0].long()].Inv() @ T[edges[:, 1].long()]).Log().tensor()
    points, pixels, ci = input                                    # single-pose reprojection
    y = T[ci.long()].Act(points)
    return -y[..., :2] / y[..., 2:] - pixels


def _same_residuals(model, input, params, shape, group, trials=2, roles=None):
    """A user module takes a fused family only if its output equals the family's residual ROW BY ROW (up to one global
    sign) at the current parameters AND at randomly perturbed ones (`roles` = (K, T, P): the BAL family).  A single scalar at a single point is not
    evidence: all-zero residuals at the start, a NaN loss, or a model that merely has the same norm there would pass
    it (ADVICE r1).  Non-finite outputs never match.  Parameters are restored exactly."""
    saved = [p.detach().clone() for p in params]
    gen = torch.Generator(device="cpu").manual_seed(20240917)
    ok = True
    try:
        with torch.no_grad():
            for trial in range(trials):
                if trial:                                         # move off the initial point (small left retraction / shift)
                    for p, s0 in zip(params, saved):
                        lie = isinstance(p, LieTensor)
                        noise = (0.05 * torch.randn(s0.shape[:-1] + (p.ltype.manifold if lie else s0.shape[-1:]),
                                                    generator=gen, dtype=torch.float64)).to(s0.device, s0.dtype)
                        new = _retract_generic(noise, s0, p.ltype) if lie else s0 + noise
                        _copy_param(p, new)
                out = model(*input)
                if not torch.is_tensor(out) or isinstance(out, LieTensor) or tuple(out.shape) != tuple(shape):
                    ok = False
                    break
                ref = _family_residuals(input, params) if roles is None else _bal_residuals(input, *roles)
                a, b = out.double(), ref.double()
                scale = 1e-4 if out.dtype == torch.float32 else 1e-9
                tol = scale * (1.0 + b.abs().max())
                err = torch.minimum((a - b).abs().max(), (a + b).abs().max())
                flag = torch.stack([(~torch.isfinite(a).all()).double(), (~torch.isfinite(b).all()).double(),
                                    (~(err <= tol)).double()]).sum().reshape(1)
                if float(_allreduce(flag, group)[0]) != 0.0:      # every rank takes the same decision
                    ok = False
                    break
    finally:
        with torch.no_grad():
            for p, s0 in zip(params, saved):
                _copy_param(p, s0)
    return ok


def _retract_generic(D, poses, ltype=SE3_type):
    """Exp(D) * poses through the LieTensor ops (any device; recognition time only)."""
    return (LieTensor(D, ltype=ltype.dual).Exp() * LieTensor(poses, ltype=ltype)).tensor()


def _is_builtin(model, cls):
    """`model` is one of this package's modules with its own forward (a subclass may add state but an overridden
    forward is a different residual and goes through signature + row-wise verification instead)."""
    return isinstance(model, cls) and type(model).forward is cls.forward


def _pgo_weight(weight, input):
    """`weight` usable by the pose-graph route: one symmetric (6,6) / (1,6,6) or per-edge (E,6,6) tensor."""
    if not (torch.is_tensor(weight) and isinstance(input, (tuple, list)) and len(input) == 2 and torch.is_tensor(input[0])):
        return False
    E = input[0].shape[0]
    if weight.dim() not in (2, 3) or tuple(weight.shape[-2:]) != (6, 6) or (weight.dim() == 3 and weight.shape[0] not in (1, E)):
        return False
    return bool(torch.allclose(weight, weight.mT))


def recognize(model, input, params, group=None, robust=(0, 1.0), solver=None, sparse=False, weight=None):
    """Return a structured problem for (model, input) or None (-> generic dense route)."""
    params = [p for p in params if p.requires_grad]
    if len(params) == 1 and getattr(params[0], 'ltype', None) is Sim3_type:
        return _recognize_lie_pgo(model, input, params, group, robust, solver, sparse, weight)
    if weight is not None and not _pgo_weight(weight, input):
        return None
    from ..module.ba import BundleAdjustment
    from .solver import CG
    if _is_builtin(model, BundleAdjustment):
        ok = (len(params) == 2 and params[0] is model.poses and params[1] is model.points_3d
              and _is_se3_param(model.poses) and (isinstance(solver, CG) or sparse)
              and model.poses.dtype in (torch.float32, torch.float64))
        if not ok:
            return None
        pix, cidx, pidx = input
        if not (_in_range(cidx, model.poses.shape[0]) and _in_range(pidx, model.points_3d.shape[0])):
            raise IndexError("BundleAdjustment: camera / point index out of range")
        tol = solver.tol if isinstance(solver, CG) else 1e-8
        maxiter = solver.maxiter if isinstance(solver, CG) else None
        return None if weight is not None else BAProblem(model, pix, cidx, pidx, _input_key(input), group, robust, tol, maxiter)
    from ..module.ba import BALBundleAdjustment
    if _is_builtin(model, BALBundleAdjustment):
        K, T, P = model.intrinsics, model.poses, model.points_3d
        ok = (len(params) == 3 and params[0] is K and params[1] is T and params[2] is P and _bal_params_ok(K, T, P)
              and (isinstance(solver, CG) or sparse) and weight is None and group is None)
        if not ok:
            return None
        pix, cidx, pidx = input
        if not (_in_range(cidx, T.shape[0]) and _in_range(pidx, P.shape[0])):
            raise IndexError("BALBundleAdjustment: camera / point index out of range")
        tol = solver.tol if isinstance(solver, CG) else 1e-8
        maxiter = solver.maxiter if isinstance(solver, CG) else None
        return BALProblem(model, pix, cidx, pidx, _input_key(input), robust, tol, maxiter, (K, T, P))
    duck = _recognize_by_signature(model, input, params, group, robust, solver, sparse, weight)
    if duck is not None:
        return duck
    if len(params) != 1 or not _is_se3_param(params[0]) or params[0].dtype not in (torch.float32, torch.float64):
        return None
    param = params[0]
    from ..module.reproj import PoseReproj
    from ..module.pgo import PoseGraph
    from .solver import CG
    from ..module.reproj import TwoPoseReproj
    if _is_builtin(model, TwoPoseReproj):
        intr = model.intr()
        if param is not model.poses or intr is None or not (isinstance(solver, CG) or sparse) or weight is not None:
            return None
        points, pixels, ia, ib = input
        if not (_in_range(ia, param.shape[0]) and _in_range(ib, param.shape[0])):
            raise IndexError("TwoPoseReproj: pose index out of range")
        tol = solver.tol if isinstance(solver, CG) else 1e-8
        maxiter = solver.maxiter if isinstance(solver, CG) else None
        return Reproj2Problem(model, points, pixels, ia, ib, intr, _input_key(input), group, robust, tol, maxiter)
    if _is_builtin(model, PoseGraph):
        # block-sparse H needs an iterative solver: taken only when the user asked for one (solver=PCG()/CG(),
        # or sparse=True as in the reference's bae route); otherwise the generic dense Cholesky route runs.
        if param is not model.nodes or not (isinstance(solver, CG) or sparse):
            return None
        edges, Z = input
        if not isinstance(Z, LieTensor) or Z.ltype is not SE3_type:
            return None
        if not _in_range(edges, param.shape[0]):
            raise IndexError("PoseGraph: edge index out of range")
        tol = solver.tol if isinstance(solver, CG) else 1e-8
        maxiter = solver.maxiter if isinstance(solver, CG) else None
        return PGOProblem(model, edges, Z, _input_key(input), group, robust, tol, maxiter, weight=weight)
    if weight is not None or (solver is not None and isinstance(solver, CG)):
        return None
    if _is_builtin(model, PoseReproj):
        if param is not model.poses:
            return None
        return ReprojProblem(model, model.prepare(*input), _input_key(input), group, robust)
    if isinstance(input, (tuple, list, dict)) or not isinstance(input, LieTensor) or input.ltype is not SE3_type:
        return None
    # record the LieTensor ops of one forward pass
    rec = []
    _lt._RECORD = rec
    try:
        with torch.no_grad():
            out = model(input)
    finally:
        _lt._RECORD = None
    if not torch.is_tensor(out) or isinstance(out, LieTensor) or len(rec) != 2:
        return None
    (op0, a, b, z), (op1, z1, _, y) = rec
    ok = (op0 == "mul" and op1 == "log" and a is param and b is input and z1 is z
          and out.data_ptr() == y.data_ptr() and out.shape == param.shape[:-1] + (6,)
          and input.shape == param.shape and not input.requires_grad and input.dtype == param.dtype
          and input.device == param.device)
    if not ok:
        return None
    return PoseInvProblem(model, param, input, _input_key(input), group, robust)
