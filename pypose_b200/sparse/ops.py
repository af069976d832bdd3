"""Block-sparse products (pypose/sparse/ops.py) on CUDA.

`bsr_bsc_matmul(A, B)` multiplies a BSR matrix by a BSC matrix on the device (csrc/bsr.cu, DESIGN.md §3.8): the output
pattern, the block products and the gradients of both values arrays are kernels, and the host reads the device twice
per product (the block-product count with the validity flag, then the number of output blocks).  `_sparse_csr_mm` is the
reference's layout dispatcher: BSR × BSC goes to `bsr_bsc_matmul`, every other pair of layouts to torch.
"""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from .. import _C

__all__ = ["bsr_bsc_matmul"]

_INT31 = 0x7fffffff


def _ws(stage, sn, nnz_a, nnz_b, T, dev):
    f = _C.lib().b200_bsr_workspace_bytes
    f.restype, f.argtypes = ctypes.c_longlong, [ctypes.c_int] + [ctypes.c_longlong] * 4
    return torch.empty(int(f(stage, sn, nnz_a, nnz_b, T)), dtype=torch.uint8, device=dev)


def _strides(v):
    return list(v.stride())


class _BsrBscValues(torch.autograd.Function):
    """Values of C = A B (and its crow / col indices) from the values and int64 indices of A (BSR) and B (BSC).  With
    vb None, B is A^T over the same storage (``A.mT``): its values are va^T and one gradient, dA + dB^T, goes to va."""

    @staticmethod
    def forward(ctx, va, vb, a_crow, a_col, b_ccol, b_row, sm, sn, sp):
        ctx.shared = vb is None
        if ctx.shared:
            vb = va.mT
        dev, dt = va.device, va.dtype
        nnz_a, dm, dn = va.shape
        nnz_b, _, dp = vb.shape
        sfx = _C.suffix(dt)
        stream = _C.stream_ptr(dev)
        T, tri, seg = 0, None, None
        ws0 = _ws(0, sn, nnz_a, nnz_b, 0, dev)
        info = torch.empty(2, dtype=torch.int64, device=dev)
        _C.check(_C.fn("b200_bsr_count")(a_crow.data_ptr(), a_col.data_ptr(), sm, nnz_a, b_ccol.data_ptr(),
                                         b_row.data_ptr(), sp, nnz_b, sn, ws0.data_ptr(), info.data_ptr(), stream),
                 "b200_bsr_count")
        T, bad = info.tolist()                               # host read 1
        if bad:
            raise ValueError("bsr_bsc_matmul: invalid index structure: the compressed pointers must run from 0 to nnz "
                             "without decreasing, and the indices must be in range and strictly increasing within "
                             "each compressed row / column")
        if T > _INT31:
            raise ValueError(f"bsr_bsc_matmul: {T} block products exceed the supported 2^31 - 1")
        if T == 0:
            crow = torch.zeros(sm + 1, dtype=torch.int64, device=dev)
            col = torch.empty(0, dtype=torch.int64, device=dev)
            out = torch.empty((0, dm, dp), dtype=dt, device=dev)
        else:
            ws1 = _ws(1, sn, nnz_a, nnz_b, T, dev)
            tri = torch.empty(T, dtype=torch.int64, device=dev)
            seg = torch.empty(T, dtype=torch.int32, device=dev)
            nnz = torch.empty(1, dtype=torch.int64, device=dev)
            _C.check(_C.fn("b200_bsr_expand")(a_col.data_ptr(), nnz_a, sm, sp, sn, nnz_b, ws0.data_ptr(), T,
                                              ws1.data_ptr(), tri.data_ptr(), seg.data_ptr(), nnz.data_ptr(), stream),
                     "b200_bsr_expand")
            del ws0
            n_c = int(nnz.item())                            # host read 2
            crow = torch.empty(sm + 1, dtype=torch.int64, device=dev)
            col = torch.empty(n_c, dtype=torch.int64, device=dev)
            out = torch.empty((n_c, dm, dp), dtype=dt, device=dev)
            sym = f"b200_bsr_numeric_{sfx}"
            _C.check(_C.fn(sym)(va.data_ptr(), *_strides(va), vb.data_ptr(), *_strides(vb), dm, dn, dp, sm, sp, T,
                                ws1.data_ptr(), tri.data_ptr(), seg.data_ptr(), n_c, crow.data_ptr(), col.data_ptr(),
                                out.data_ptr(), stream), sym)
        ctx.mark_non_differentiable(crow, col)
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            ctx.save_for_backward(va, None if ctx.shared else vb, tri, seg)
        ctx.T = T
        return out, crow, col

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, _g_crow, _g_col):
        va, vb, tri, seg = ctx.saved_tensors
        need_a, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if ctx.shared:
            vb, need_b = va.mT, need_a
        nnz_a, dm, dn = va.shape
        nnz_b, _, dp = vb.shape
        ga = torch.zeros_like(va, memory_format=torch.contiguous_format) if need_a else None
        gb = torch.zeros_like(vb, memory_format=torch.contiguous_format) if need_b else None
        if ctx.T == 0 or g_out is None:
            return ga, None if ctx.shared else gb, None, None, None, None, None, None, None
        dev = va.device
        g = g_out.to(va.dtype).contiguous()
        ws = _ws(2, 0, nnz_a, nnz_b, ctx.T, dev)
        sym = f"b200_bsr_grad_{_C.suffix(va.dtype)}"
        _C.check(_C.fn(sym)(va.data_ptr(), *_strides(va), vb.data_ptr(), *_strides(vb), g.data_ptr(), dm, dn, dp,
                            tri.data_ptr(), seg.data_ptr(), ctx.T, nnz_a, nnz_b, ws.data_ptr(),
                            ga.data_ptr() if need_a else None, gb.data_ptr() if need_b else None,
                            _C.stream_ptr(dev)), sym)
        if ctx.shared:
            return ga + gb.mT if need_a else None, None, None, None, None, None, None, None, None
        return ga, gb, None, None, None, None, None, None, None


def _check(bsr, bsc):
    """(m, n, p, dm, dn, dp) of a valid BSR × BSC pair; raises otherwise."""
    for name, t in (("bsr", bsr), ("bsc", bsc)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"bsr_bsc_matmul: {name} must be a tensor, got {type(t).__name__}")
    if bsr.layout == torch.sparse_bsc and bsc.layout == torch.sparse_bsr:
        raise NotImplementedError("bsr_bsc_matmul: bsc × bsr is not implemented; pass a torch.sparse_bsr first operand "
                                  "and a torch.sparse_bsc second operand")
    if bsr.layout != torch.sparse_bsr or bsc.layout != torch.sparse_bsc:
        raise ValueError(f"bsr_bsc_matmul: expected torch.sparse_bsr × torch.sparse_bsc, got {bsr.layout} × {bsc.layout}")
    if bsr.dim() != 2 or bsc.dim() != 2 or bsr.values().dim() != 3 or bsc.values().dim() != 3:
        raise ValueError("bsr_bsc_matmul: bsr and bsc must be 2-dimensional (batch and dense dimensions are not "
                         f"supported), got shapes {tuple(bsr.shape)} and {tuple(bsc.shape)}")
    if bsr.dtype != bsc.dtype:
        raise ValueError(f"bsr_bsc_matmul: both operands must have one dtype, got {bsr.dtype} and {bsc.dtype}")
    if bsr.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"bsr_bsc_matmul: float32 and float64 are supported, got {bsr.dtype}")
    (m, n), (n2, p) = bsr.shape, bsc.shape
    (dm, dn), (dn2, dp) = bsr.values().shape[1:], bsc.values().shape[1:]
    if n != n2:
        raise ValueError(f"bsr_bsc_matmul: inner sizes differ, {tuple(bsr.shape)} × {tuple(bsc.shape)}")
    if dn != dn2:
        raise ValueError(f"bsr_bsc_matmul: inner block sizes differ, ({dm}, {dn}) blocks × ({dn2}, {dp}) blocks")
    if min(dm, dn, dp) < 1 or m % dm or n % dn or p % dp:
        raise ValueError(f"bsr_bsc_matmul: shapes {tuple(bsr.shape)} and {tuple(bsc.shape)} are not divisible by the "
                         f"blocks ({dm}, {dn}) and ({dn2}, {dp})")
    for t in (bsr, bsc):
        if not t.is_cuda:
            raise NotImplementedError(f"bsr_bsc_matmul: expected CUDA tensors (no CPU path), got {t.device}")
    if bsr.device != bsc.device:
        raise ValueError(f"bsr_bsc_matmul: both operands must be on one device, got {bsr.device} and {bsc.device}")
    return m, n, p, dm, dn, dp


def _is_transpose_of(bsc, bsr):
    """Whether bsc is bsr.mT: the same index and value storage, read transposed, and, when either carries gradients,
    bsc produced from bsr by the transpose on the autograd graph (so ``bsr.detach().mT`` or a new tensor over the same
    storage is not taken for it, and each operand keeps its own gradient)."""
    va, vb = bsr.values(), bsc.values()
    if not (bsc.ccol_indices().data_ptr() == bsr.crow_indices().data_ptr() and
            bsc.row_indices().data_ptr() == bsr.col_indices().data_ptr() and vb.data_ptr() == va.data_ptr() and
            vb.shape == va.mT.shape and vb.stride() == va.mT.stride()):
        return False
    if not bsr.requires_grad and not bsc.requires_grad:
        return True
    f = bsc.grad_fn
    if f is None or not type(f).__name__.startswith("TransposeBackward") or len(f.next_functions) != 1:
        return False
    node = f.next_functions[0][0]
    if bsr.grad_fn is not None:
        return node is bsr.grad_fn
    return type(node).__name__ == "AccumulateGrad" and node.variable is bsr


def bsr_bsc_matmul(bsr, bsc):
    r"""The product C = A B of a block-sparse row matrix A and a block-sparse column matrix B.

    Args:
        bsr (torch.Tensor): A, a 2-D ``torch.sparse_bsr`` tensor of size (m, n) with (dm, dn) blocks.
        bsc (torch.Tensor): B, a 2-D ``torch.sparse_bsc`` tensor of size (n, p) with (dn, dp) blocks.

    Returns:
        torch.Tensor: C, a ``torch.sparse_bsr`` tensor of size (m, p) with (dm, dp) blocks and int64 indices, on the
        inputs' device and in their dtype.  Block (i, j) is stored exactly when block row i of A and block column j of B
        share a stored block index k, explicitly stored zero blocks included; columns are sorted within each row.

    Either index dtype (int32 or int64) is accepted for each input, and values may be non-contiguous, so ``A @ A.mT``
    is ``bsr_bsc_matmul(A, A.mT)`` without a copy.  Gradients flow to the values of both operands (through
    ``torch.sparse_bsr_tensor(..., values)`` / ``.values()``); the gradients are bit-reproducible.  When B is ``A.mT``
    (it shares A's index and value storage and was made from A by the transpose on the autograd graph), A's values are
    taken once and receive dA + dB^T in one gradient; ``A.detach().mT`` or ``A.mT`` with ``A.detach()`` first keep
    separate gradients.  The
    gradient kernels need no host reads, but torch's own backward of ``torch.sparse_bsr_tensor`` / ``.values()`` forms
    dense (m, n) tensors, so gradients through the sparse constructors are practical only for small matrices.

    Differences from the reference:

    * CPU tensors raise ``NotImplementedError``: there is no CPU path.
    * The indices must be in range and strictly increasing within each compressed row or column, and the compressed
      pointers must run from 0 to nnz without decreasing (torch's invariants).  A violation raises ``ValueError``.
    * More than 2^31 - 1 block products raise ``ValueError``.
    * ``bsc × bsr`` raises ``NotImplementedError`` (the reference raises ``TypeError``), other layouts, batch or dense
      dimensions, mixed dtypes and shapes that do not divide into the blocks raise ``ValueError``.
    * The result carries gradients.

    Example:
        >>> A = torch.sparse_bsr_tensor(crow, col, values, size=(12, 18)).cuda()   # (3, 6) blocks
        >>> C = pp.bsr_bsc_matmul(A, A.mT)                                          # (12, 12), (3, 3) blocks
    """
    m, n, p, dm, dn, dp = _check(bsr, bsc)
    sm, sn, sp = m // dm, n // dn, p // dp
    va, vb = bsr.values(), bsc.values()
    dev = va.device
    if min(sm, sn, sp) == 0:
        return torch.sparse_bsr_tensor(torch.zeros(sm + 1, dtype=torch.int64, device=dev),
                                       torch.empty(0, dtype=torch.int64, device=dev),
                                       torch.zeros((0, dm, dp), dtype=va.dtype, device=dev), size=(m, p),
                                       check_invariants=False)
    idx = [t.to(torch.int64).contiguous() for t in (bsr.crow_indices(), bsr.col_indices(), bsc.ccol_indices(),
                                                    bsc.row_indices())]
    if idx[0].numel() != sm + 1 or idx[2].numel() != sp + 1 or idx[1].numel() != va.shape[0] or \
            idx[3].numel() != vb.shape[0]:
        raise ValueError("bsr_bsc_matmul: the index arrays do not match the shapes and the stored blocks")
    if max(sm, sn, sp) > _INT31:
        raise ValueError(f"bsr_bsc_matmul: block grids of more than 2^31 - 1 rows or columns are not supported, got "
                         f"({sm}, {sn}) × ({sn}, {sp}) blocks")
    if va.shape[0] > _INT31 or vb.shape[0] > _INT31:
        raise ValueError("bsr_bsc_matmul: more than 2^31 - 1 stored blocks in an operand")
    # B = A.mT (A's index and value storage, and A's autograd path): pass A's values once, so that autograd does not
    # have to add two sparse gradients of A (torch has no CUDA kernel for adding BSR tensors)
    shared = _is_transpose_of(bsc, bsr)
    with torch.cuda.device(dev):
        values, crow, col = _BsrBscValues.apply(va, None if shared else vb, *idx, sm, sn, sp)
        return torch.sparse_bsr_tensor(crow, col, values, size=(m, p), check_invariants=False)


def _sparse_csr_mm(mat1, mat2):
    """mat1 @ mat2 for compressed sparse layouts, routed as the reference routes them.

    BSR × BSC runs :func:`bsr_bsc_matmul` (so it needs CUDA tensors); BSC × BSR raises ``NotImplementedError``.
    CSR × CSR is ``torch.addmm`` onto a CSR zero; CSR / CSC pairs are converted to CSR first; CSC × strided converts the
    CSC operand to CSR; any × strided is ``torch.addmm`` onto a strided zero; every other pair is ``torch.addmm`` onto a
    zero of mat1's layout (the reference passes a one-element tuple there and raises ``TypeError``).
    """
    l1, l2 = mat1.layout, mat2.layout
    if l1 == torch.sparse_bsr and l2 == torch.sparse_bsc:
        return bsr_bsc_matmul(mat1, mat2)
    if l1 == torch.sparse_bsc and l2 == torch.sparse_bsr:
        raise NotImplementedError("_sparse_csr_mm: bsc × bsr is not implemented")
    size = (mat1.shape[0], mat2.shape[1])
    compressed = (torch.sparse_csr, torch.sparse_csc)
    if l1 == torch.sparse_csr and l2 == torch.sparse_csr:
        zero = torch.zeros(size, dtype=mat2.dtype, device=mat2.device, layout=torch.sparse_csr)
        return torch.addmm(zero, mat1, mat2, beta=0.0, alpha=1.0)
    if l1 in compressed and l2 in compressed:
        return _sparse_csr_mm(mat1.to_sparse_csr(), mat2.to_sparse_csr())
    if l1 == torch.sparse_csc and l2 == torch.strided:
        return _sparse_csr_mm(mat1.to_sparse_csr(), mat2)
    if l2 == torch.strided:
        zero = torch.zeros(size, dtype=mat1.dtype, device=mat1.device)
        return torch.addmm(zero, mat1, mat2, beta=0.0, alpha=1.0)
    zero = torch.zeros(size, dtype=mat1.dtype, device=mat1.device, layout=l1)
    return torch.addmm(zero, mat1, mat2, beta=0.0, alpha=1.0)
