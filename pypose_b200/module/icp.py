"""Batched point-to-point ICP (reference: pypose/module/icp.py) on the kernels of csrc/knn.cu."""
import ctypes
import math

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from .. import _C
from ..function.geometry import _ORD, _pc_batch
from ..lietensor import LieTensor, SE3_type
from ..utils.stepper import ReduceToBason

_CHUNKS = (4, 8, 16, 32)      # iterations enqueued per host read of the device-decided loop


def _check_se3(T, what):
    if T is not None and not (isinstance(T, LieTensor) and isinstance(T.ltype, type(SE3_type))):
        raise TypeError(f"ICP: {what} must be an SE3 LieTensor, got {type(T).__name__}"
                        + (f" of type {T.ltype}" if isinstance(T, LieTensor) else ""))


def _init_rows(init, batch, device, dtype):
    """The initial SE3 as (1 | prod(batch), 7) contiguous rows on `device` in `dtype` (None: identity).  An init on
    another device (a CPU `pp.identity_SE3(B)`, say) is copied over here, before any pointer reaches the kernels."""
    if init is None:
        return None
    it = init.tensor().detach().to(device=device, dtype=dtype)
    if math.prod(init.shape[:-1]) == 1:
        return it.reshape(1, 7).contiguous()
    return it.expand(*batch, 7).reshape(math.prod(batch), 7).contiguous()


class ICP(nn.Module):
    """Iterative Closest Point: the SE3 `T` that moves `source` (..., Ns, 3) onto `target` (..., Nt, 3).

    Each iteration matches every point of `A source` to its nearest point of `target` (`ord`-norm), takes the mean
    nearest distance as the loss, solves the Kabsch step `T` of the matched pairs, composes `A <- T A` and hands the loss
    to `stepper.step` (the reference's order: match, error, Kabsch, apply, step).  `A` starts at `init` (or the identity).

    * Batch dimensions of source, target and init broadcast; source and target may have different point counts.
    * The default stepper is `pp.utils.ReduceToBason(steps=200)`.  With a non-verbose `ReduceToBason` the stop rule runs on
      the GPU and the host reads the state once per chunk of iterations; afterwards the stepper holds the `steps`, `last`,
      `patience_count` and `continual()` the host loop would have left.  Any other stepper is called every iteration.
    * Returns the composed `A` (an SE3 LieTensor of the broadcast batch).  The reference returns `svdtf(source, A source)`,
      the same transform up to rounding when the source is not degenerate.
    * The Kabsch step is solved in fp64 with a defined answer for rank-deficient (planar, collinear, coincident) matches
      (DESIGN.md §3.4).  CUDA tensors only.
    * Gradients: when autograd is on and `source`, `target` or `init` requires grad, the forward also records each
      iteration's matches and the backward runs the reference's graph (knn -> gather -> svdtf -> Act per iteration, closed
      by svdtf(source, A source)) in reverse on the GPU, with matches and iteration count held fixed.  The returned
      transform is bit-identical to the call without grad.  Rank-deficient Kabsch steps have defined gradients (DESIGN.md
      §3.4); there is no double backward."""

    def __init__(self, init=None, stepper=None):
        super().__init__()
        _check_se3(init, "init")
        self.init = init
        self.stepper = stepper if stepper is not None else ReduceToBason(steps=200)
        self._host = None

    def forward(self, source, target, ord=2, dim=-1, init=None):
        if init is None:
            init = self.init
        _check_se3(init, "init")
        source = source.tensor() if isinstance(source, LieTensor) else source
        target = target.tensor() if isinstance(target, LieTensor) else target
        if not source.is_cuda or not target.is_cuda:
            raise NotImplementedError(f"ICP: expected CUDA tensors (no CPU path), got {source.device} / {target.device}")
        if source.device != target.device or source.dtype != target.dtype:
            raise ValueError("ICP: source and target must share device and dtype")
        sfx = _C.suffix(source.dtype)
        if dim not in (-1, source.dim() - 1) or source.shape[-1] != 3 or target.shape[-1] != 3:
            raise ValueError("ICP: points must be (..., N, 3) with the coordinates in the last dimension")
        if ord not in _ORD:
            raise ValueError(f"ICP: ord must be 1, 2 or inf, got {ord}")
        Ns, Nt = source.shape[-2], target.shape[-2]
        if Ns < 1 or Nt < 1:
            raise ValueError("ICP: source and target need at least one point each")
        shapes = [source.shape[:-2], target.shape[:-2]] + ([init.shape[:-1]] if init is not None else [])
        batch = torch.broadcast_shapes(*shapes)
        B = math.prod(batch)
        dev, dtype = source.device, source.dtype
        out = torch.empty(*batch, 7, dtype=dtype, device=dev)
        if B == 0:
            return LieTensor(out, ltype=SE3_type)
        grad = torch.is_grad_enabled() and (source.requires_grad or target.requires_grad
                                             or (init is not None and init.requires_grad))
        if grad:
            src, tgt = _pc_batch(source, target, batch)
            it = None if init is None else _init_rows_grad(init, batch, dev, dtype)
            out = _ICPFn.apply(src, tgt, it, self, ord, batch, Ns, Nt)
            return LieTensor(out.view(*batch, 7), ltype=SE3_type)
        src, tgt = _pc_batch(source.detach(), target.detach(), batch)
        it = _init_rows(init, batch, dev, dtype)
        self._run(src, tgt, it, out, ord, batch, B, Ns, Nt)
        return LieTensor(out, ltype=SE3_type)

    def _run(self, src, tgt, it, out, ord, batch, B, Ns, Nt, traces=None):
        """The iterations on the GPU; `out` gets A.  traces (a list): record every iteration, appending (trace tensor,
        iterations it holds) per call.  Returns the workspace (it holds A in fp64) and the number of iterations run."""
        dev, dtype = src.device, src.dtype
        sfx = _C.suffix(dtype)
        q = _C.lib().b200_icp_workspace_bytes
        q.restype, q.argtypes = ctypes.c_longlong, [ctypes.c_longlong] * 2
        with torch.cuda.device(dev):
            ws = torch.empty(int(q(B, Ns)), dtype=torch.uint8, device=dev)
            last = torch.empty(B, dtype=dtype, device=dev)
            sym = f"b200_icp_{sfx}" if traces is None else f"b200_icp_rec_{sfx}"
            f = _C.fn(sym)
            if traces is not None:
                tq = _C.lib().b200_icp_trace_bytes
                tq.restype, tq.argtypes = ctypes.c_longlong, [ctypes.c_longlong] * 3

                def rec(n):
                    t = torch.empty(int(tq(B, Ns, n)), dtype=torch.uint8, device=dev)
                    traces.append((t, n))
                    return (t.data_ptr(),)
            else:
                def rec(n):
                    return ()
            st = self.stepper
            device_rule = type(st) is ReduceToBason and not st.verbose
            common = (src.data_ptr(), src.shape[1] * 3 if src.shape[0] > 1 else 0,
                      tgt.data_ptr(), tgt.shape[1] * 3 if tgt.shape[0] > 1 else 0,
                      it.data_ptr() if it is not None else None, 7 if it is not None and it.shape[0] > 1 else 0,
                      out.data_ptr())
            st.reset()
            if device_rule:
                err = torch.empty(B, dtype=dtype, device=dev)
                if self._host is None:
                    self._host = torch.zeros(8, dtype=torch.float64).pin_memory()
                    self._seq = 0
                ctl = (int(st.max_steps), int(st.patience), float(st.decreasing), float(st.tol))
                first, n = 1, 0
                while True:
                    chunk = _CHUNKS[min(n, len(_CHUNKS) - 1)]
                    self._seq += 1
                    _C.check(f(*common, err.data_ptr(), last.data_ptr(), ws.data_ptr(), B, Ns, Nt, _ORD[ord], first,
                               chunk, 1, *ctl, self._host.data_ptr(), self._seq, *rec(chunk), _C.stream_ptr(dev)), sym)
                    first, n = 0, n + 1
                    h = self._host.tolist()
                    if h[2] == 0.0:
                        break
                st.steps, st.patience_count, st._continual = int(h[0]), int(h[1]), False
                st.last = last.view(batch)
                ran = st.steps
            else:
                first, ran = 1, 0
                while st.continual():
                    err = torch.empty(B, dtype=dtype, device=dev)
                    _C.check(f(*common, err.data_ptr(), last.data_ptr(), ws.data_ptr(), B, Ns, Nt, _ORD[ord], first, 1, 0,
                               0, 0, 0.0, 0.0, None, 0, *rec(1), _C.stream_ptr(dev)), sym)
                    first, ran = 0, ran + 1
                    st.step(err.view(batch))
        return ws, ran


def _init_rows_grad(init, batch, device, dtype):
    """_init_rows on the autograd graph: (1 | prod(batch), 7) rows whose gradient reaches `init`."""
    it = init.tensor().to(device=device, dtype=dtype)
    if math.prod(init.shape[:-1]) == 1:
        return it.reshape(1, 7).contiguous()
    return it.expand(*batch, 7).reshape(math.prod(batch), 7).contiguous()


class _ICPFn(torch.autograd.Function):
    """ICP with a recorded trace; backward: b200_icp_bwd (csrc/knn.cu).  src (1|B, Ns, 3), tgt (1|B, Nt, 3),
    init (1|B, 7) or None; returns (B, 7)."""

    @staticmethod
    def forward(ctx, src, tgt, init, icp, ord, batch, Ns, Nt):
        B = math.prod(batch)
        out = torch.empty(B, 7, dtype=src.dtype, device=src.device)
        traces = []
        ws, K = icp._run(src, tgt, init, out, ord, batch, B, Ns, Nt, traces)
        addrs = [t.data_ptr() + j * (t.numel() // n) for t, n in traces for j in range(n)][:K]
        ctx.save_for_backward(src, tgt, init)
        ctx.keep = (ws, traces, addrs, B, Ns, Nt)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        src, tgt, init = ctx.saved_tensors
        ws, traces, addrs, B, Ns, Nt = ctx.keep
        dev, dtype = src.device, src.dtype
        need = ctx.needs_input_grad
        gs = torch.empty_like(src) if need[0] else None
        gt = torch.empty_like(tgt) if need[1] else None
        gi = torch.empty_like(init) if init is not None and need[2] else None
        q = _C.lib().b200_icp_bwd_workspace_bytes
        q.restype, q.argtypes = ctypes.c_longlong, [ctypes.c_longlong] * 4
        with torch.cuda.device(dev):
            bws = torch.empty(int(q(B, Ns, Nt, tgt.shape[0])), dtype=torch.uint8, device=dev)
            g = gout.to(dtype).contiguous()
            sym = f"b200_icp_bwd_{_C.suffix(dtype)}"
            K = len(addrs)
            arr = (ctypes.c_longlong * max(K, 1))(*addrs)
            ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
            _C.check(_C.fn(sym)(src.data_ptr(), Ns * 3 if src.shape[0] > 1 else 0, tgt.data_ptr(),
                                Nt * 3 if tgt.shape[0] > 1 else 0, ptr(init), 7 if init is not None and init.shape[0] > 1 else 0,
                                ws.data_ptr(), arr, K, g.data_ptr(), ptr(gs), ptr(gt), ptr(gi), bws.data_ptr(), B, Ns, Nt,
                                _C.stream_ptr(dev)), sym)
        return gs, gt, gi, None, None, None, None, None
