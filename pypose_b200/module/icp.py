"""Batched point-to-point ICP (reference: pypose/module/icp.py) on the kernels of csrc/knn.cu."""
import ctypes
import math

import torch
from torch import nn

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
      (DESIGN.md §3.4).  CUDA tensors only; there is no autograd through ICP."""

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
        src, tgt = _pc_batch(source.detach(), target.detach(), batch)
        it = _init_rows(init, batch, dev, dtype)
        q = _C.lib().b200_icp_workspace_bytes
        q.restype, q.argtypes = ctypes.c_longlong, [ctypes.c_longlong] * 2
        with torch.cuda.device(dev):
            ws = torch.empty(int(q(B, Ns)), dtype=torch.uint8, device=dev)
            last = torch.empty(B, dtype=dtype, device=dev)
            sym = f"b200_icp_{sfx}"
            f = _C.fn(sym)
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
                               chunk, 1, *ctl, self._host.data_ptr(), self._seq, _C.stream_ptr(dev)), sym)
                    first, n = 0, n + 1
                    h = self._host.tolist()
                    if h[2] == 0.0:
                        break
                st.steps, st.patience_count, st._continual = int(h[0]), int(h[1]), False
                st.last = last.view(batch)
            else:
                first = 1
                while st.continual():
                    err = torch.empty(B, dtype=dtype, device=dev)
                    _C.check(f(*common, err.data_ptr(), last.data_ptr(), ws.data_ptr(), B, Ns, Nt, _ORD[ord], first, 1, 0,
                               0, 0, 0.0, 0.0, None, 0, _C.stream_ptr(dev)), sym)
                    first = 0
                    st.step(err.view(batch))
        return LieTensor(out, ltype=SE3_type)
