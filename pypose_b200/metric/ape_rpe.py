"""Trajectory metrics: absolute and relative pose error (pypose/metric/ape_rpe.py) on CUDA.

Every step that grows with the trajectory runs in csrc/traj.cu (DESIGN.md §3.6): timestamp association, the path walk of
distance pairing, the per-pair errors and the statistics.  Torch is used for memory, index gathers and the alignment
(`svdstf` on the associated translations, or r_0 e_0^-1).  All arithmetic is fp64, as the reference's StampedSE3 does;
fp32 poses are widened inside the kernels and fp32 stamps by `.to(float64)`.
"""
import ctypes
import warnings

import torch

from .. import _C
from ..function.geometry import svdstf, _check_cuda
from ..lietensor import LieTensor, SE3, SE3_type

_ETYPES = {'translation': 0, 'rotation': 1, 'pose': 2, 'radian': 3, 'degree': 4}
_KEYS = ['Max', 'Min', 'Mean', 'Median', 'RMSE', 'SSE', 'STD']
_OTYPES = ['All'] + _KEYS


def _poses(name, pose):
    if not (isinstance(pose, LieTensor) and isinstance(pose.ltype, type(SE3_type))):
        raise ValueError(f"{name}: the poses must be an SE3 LieTensor")
    t = pose.tensor()
    if t.dim() != 2 or t.shape[-1] != 7 or t.shape[0] == 0:
        raise ValueError(f"{name}: expected one non-empty trajectory of shape (N, 7), got {tuple(t.shape)}")
    _check_cuda(name, t)
    return t


def _stamps(name, stamp, n, dev):
    if stamp is None:
        return torch.arange(n, dtype=torch.float64, device=dev)
    s = torch.as_tensor(stamp)
    if s.dim() != 1 or s.shape[0] != n:
        raise ValueError(f"{name}: timestamps and poses must have the same length, got {tuple(s.shape)} for {n} poses")
    return s.to(device=dev, dtype=torch.float64).contiguous()   # a new tensor unless it already is: never written


def _ws(n, dev):
    f = _C.lib().b200_traj_workspace_bytes
    f.restype, f.argtypes = ctypes.c_longlong, [ctypes.c_longlong]
    return torch.empty(int(f(int(n))), dtype=torch.uint8, device=dev)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _associate(name, rstamp, rpose, estamp, epose, diff, offset, thresh):
    """Associated row indices (r_idx, e_idx) of both trajectories and their pose tensors; one host read."""
    rt, et = _poses(name, rpose), _poses(name, epose)
    if rt.device != et.device:
        raise ValueError(f"{name}: both trajectories must be on one device, got {rt.device} and {et.device}")
    if rt.dtype != et.dtype:            # one kernel flavour reads both: widen the fp32 one, exactly
        rt, et = rt.double(), et.double()
    dev = rt.device
    rs, es = _stamps(name, rstamp, rt.shape[0], dev), _stamps(name, estamp, et.shape[0], dev)
    snd_longer = es.shape[0] > rs.shape[0]
    short, long_ = (rs, es) if snd_longer else (es, rs)
    off = float(offset) if snd_longer else -float(offset)
    ns = short.shape[0]
    ws = _ws(ns, dev)
    idx_s = torch.empty(ns, dtype=torch.long, device=dev)
    idx_l = torch.empty(ns, dtype=torch.long, device=dev)
    info = torch.empty(3, dtype=torch.long, device=dev)
    _C.check(_C.fn("b200_traj_match")(short.data_ptr(), ns, long_.data_ptr(), long_.shape[0], off, float(diff),
                                      ws.data_ptr(), idx_s.data_ptr(), idx_l.data_ptr(), info.data_ptr(),
                                      _C.stream_ptr(dev)), "b200_traj_match")
    cnt, bad_s, bad_l = info.tolist()
    if bad_s or bad_l:
        raise ValueError(f"{name}: timestamps must be ascending (non-decreasing, no NaN)")
    if cnt == 0:
        raise ValueError(f"{name}: found no matching timestamps between estimation and reference with max time diff "
                         f"{diff} (s) and time offset {offset} (s)")
    if cnt < thresh * ns:
        warnings.warn("The estimated trajectory has not enough timestamps within the GT timestamps. "
                      "May be not be enough for aligned and not accurate results.", category=Warning, stacklevel=3)
    idx_s, idx_l = idx_s[:cnt], idx_l[:cnt]
    r_idx, e_idx = (idx_s, idx_l) if snd_longer else (idx_l, idx_s)
    return rt, et, r_idx, e_idx


def _alignment(name, rt, et, r_idx, e_idx, align, scale, nposes, origin):
    """The Sim3 [t, q, s] (fp64, device) applied to the estimate, or None for the identity."""
    if align or scale:
        if nposes == -1:
            m = r_idx.shape[0]
        elif isinstance(nposes, int) and nposes >= 1:
            m = min(nposes, r_idx.shape[0])
        else:
            raise ValueError(f"{name}: nposes must be -1 or a positive int, got {nposes}")
        est = et[e_idx[:m], :3].double()
        ref = rt[r_idx[:m], :3].double()
        return svdstf(est, ref, scale).tensor().double().reshape(8).contiguous()
    if origin:
        r0 = SE3(rt.index_select(0, r_idx[:1]).double())
        e0 = SE3(et.index_select(0, e_idx[:1]).double())
        T = (r0 @ e0.Inv()).tensor().reshape(7)
        return torch.cat((T, T.new_ones(1))).contiguous()
    return None


def _errors(rt, et, ra, rb, ea, eb, S, etype):
    M = ra.shape[0]
    err = torch.empty(M, dtype=torch.float64, device=rt.device)
    sym = f"b200_traj_err_{_C.suffix(rt.dtype)}"
    _C.check(_C.fn(sym)(rt.data_ptr(), rt.stride(0), rt.stride(1), et.data_ptr(), et.stride(0), et.stride(1),
                        ra.data_ptr(), _ptr(rb), ea.data_ptr(), _ptr(eb), _ptr(S), M, _ETYPES[etype], err.data_ptr(),
                        _C.stream_ptr(rt.device)), sym)
    return err


def _statistics(err, otype):
    dev = err.device
    out = torch.empty(7, dtype=torch.float64, device=dev)
    mask = 0x7f if otype == 'All' else 1 << _KEYS.index(otype)
    ws = _ws(0, dev)
    _C.check(_C.fn("b200_traj_stats")(err.data_ptr(), err.shape[0], mask, ws.data_ptr(), out.data_ptr(),
                                      _C.stream_ptr(dev)), "b200_traj_stats")
    if otype == 'All':
        return {k: out[i] for i, k in enumerate(_KEYS)}
    return out[_KEYS.index(otype)]


def _check_types(etype, otype):
    if etype not in _ETYPES:
        raise ValueError(f"Unknown output type: {etype}")
    if otype not in _OTYPES:
        raise ValueError(f"Unknown output metric type, select one in {_OTYPES}")


def _pairs_by_dist(rt, idx, S, delta, tol, all):
    """pairs_by_dist on the rows `idx` of `rt` aligned by S: (src, tgt) positions in idx; one host read."""
    n = idx.shape[0]
    dev = rt.device
    ws = _ws(n, dev)
    src = torch.empty(n, dtype=torch.long, device=dev)
    tgt = torch.empty(n, dtype=torch.long, device=dev)
    cnt = torch.empty(1, dtype=torch.long, device=dev)
    sym = f"b200_traj_pairs_dist_{_C.suffix(rt.dtype)}"
    _C.check(_C.fn(sym)(rt.data_ptr(), rt.stride(0), rt.stride(1), idx.data_ptr(), n, _ptr(S), float(delta), float(tol),
                        int(bool(all)), ws.data_ptr(), src.data_ptr(), tgt.data_ptr(), cnt.data_ptr(),
                        _C.stream_ptr(dev)), sym)
    c = int(cnt.item())
    if all:
        return src[:c], tgt[:c]
    lst = src[:c]
    return lst[:-1], lst[1:]


def _pairs_by_frames(n, delta, all, dev):
    d = int(delta)
    if d < 1:
        raise ValueError("delta must >= 1")
    if all:
        src = torch.arange(max(n - d, 0), dtype=torch.long, device=dev)
        return src, src + d
    ids = torch.arange(0, n, d, dtype=torch.long, device=dev)
    return ids[:-1], ids[1:]


def ape(rstamp, rpose, estamp, epose, etype: str = "translation", diff: float = 0.01,
        offset: float = 0.0, align: bool = False, scale: bool = False, nposes: int = -1,
        origin: bool = False, thresh: float = 0.3, otype: str = 'All'):
    r'''Absolute Pose Error (APE) between two trajectories, as ``pypose.metric.ape``.

    Args:
        rstamp (``Tensor`` or ``None``): (N_r) timestamps of the reference; ``None``: 0, 1, 2, ...
        rpose (``LieTensor``): (N_r, 7) SE3 reference poses, fp32 or fp64, on CUDA.
        estamp (``Tensor`` or ``None``): (N_e) timestamps of the estimate.
        epose (``LieTensor``): (N_e, 7) SE3 estimated poses on the same device.
        etype (``str``): ``'translation'`` :math:`\|t_e - t_r\|`, ``'rotation'`` :math:`\|R_e^T R_r - I_3\|_F`,
            ``'pose'`` :math:`\|T_e^{-1} T_r - I_4\|_F`, ``'radian'`` :math:`\|\mathrm{Log}(R_e^T R_r)\|` or
            ``'degree'`` (the same in degrees).  Default ``'translation'``.
        diff (``float``): the largest time difference (exclusive) of an associated pair.  Default 0.01.
        offset (``float``): time offset added to the stamps of the longer trajectory (negated when that is the
            reference).  Default 0.0.
        align (``bool``): align the estimate by ``svdstf`` of the associated translations.  Default False.
        scale (``bool``): also correct the scale (implies ``align``).  Default False.
        nposes (``int``): align on the first ``nposes`` associated poses; -1 for all.  Default -1.
        origin (``bool``): without ``align``/``scale``, align by the first poses: :math:`r_0 e_0^{-1}`.
        thresh (``float``): warn when fewer than ``thresh`` times the shorter trajectory's poses are associated.
        otype (``str``): ``'All'`` or one of ``'Max'``, ``'Min'``, ``'Mean'``, ``'Median'``, ``'RMSE'``, ``'SSE'``,
            ``'STD'``.  Default ``'All'``.

    Returns:
        ``dict`` of 0-dim fp64 tensors with the keys Max, Min, Mean, Median, RMSE, SSE, STD (in that order) for
        ``otype='All'``, otherwise that one 0-dim fp64 tensor, on the poses' device.  The median is the lower median.

    Differences from the reference:
        - ``nposes`` means the first ``nposes`` poses (the reference slices coordinates instead, so it has no effect).
        - The caller's stamps are never shifted by ``offset``.
        - Invalid input (unsorted stamps, mismatched lengths, no match) raises ``ValueError`` instead of failing an
          ``assert``.  CPU poses raise ``NotImplementedError``: there is no CPU path.
        - Association takes O(N log N) work and no (N_short, N_long) matrix, and reads the host once.
    '''
    _check_types(etype, otype)
    rt, et, r_idx, e_idx = _associate("ape", rstamp, rpose, estamp, epose, diff, offset, thresh)
    S = _alignment("ape", rt, et, r_idx, e_idx, align, scale, nposes, origin)
    return _statistics(_errors(rt, et, r_idx, None, e_idx, None, S, etype), otype)


def rpe(rstamp, rpose, estamp, epose, etype: str = "translation", diff: float = 0.01,
        offset: float = 0.0, align: bool = False, scale: bool = False, nposes: int = -1,
        origin: bool = False, associate: str = 'frame', delta: float = 1.0, rtol: float = 0.1,
        all: bool = False, thresh: float = 0.3, rpair: bool = False, otype: str = 'All'):
    r'''Relative Pose Error (RPE) between two trajectories, as ``pypose.metric.rpe``.

    Takes the arguments of :func:`ape` and:

    Args:
        associate (``str``): ``'frame'`` pairs poses ``delta`` frames apart, ``'distance'`` pairs them ``delta``
            apart along the path.  Default ``'frame'``.
        delta (``float``): the pair interval in frames or in path length.  Default 1.0.
        rtol (``float``): with ``'distance'`` and ``all``, accept a pair whose path length is within ``delta * rtol``
            of ``delta``.  Default 0.1.
        all (``bool``): use every pose as a pair source (otherwise consecutive, non-overlapping pairs).
        rpair (``bool``): choose the pairs on the reference path instead of the aligned estimate.

    The error of a pair (a, b) is that of :math:`E = (r_a^{-1} r_b)^{-1} (e_a^{-1} e_b)`; ``'translation'`` is
    :math:`\|t(E)\|`.  Returns as :func:`ape`.

    Differences from the reference:
        - Those of :func:`ape`.
        - Distance pairing runs on CUDA: one sequential walk over the path in one CTA and a binary search per pose,
          with the reference's rounding, so the pair sets are the reference's.  It reads the host once more.
        - An empty pair list raises ``ValueError`` (the reference fails later, inside StampedSE3).
    '''
    _check_types(etype, otype)
    if associate not in ('frame', 'distance'):
        raise ValueError(f"unsupported delta unit: {associate}")
    rt, et, r_idx, e_idx = _associate("rpe", rstamp, rpose, estamp, epose, diff, offset, thresh)
    S = _alignment("rpe", rt, et, r_idx, e_idx, align, scale, nposes, origin)
    if associate == 'frame':
        src, tgt = _pairs_by_frames(r_idx.shape[0], delta, all, rt.device)
    elif rpair:
        src, tgt = _pairs_by_dist(rt, r_idx, None, delta, delta * rtol, all)
    else:
        src, tgt = _pairs_by_dist(et, e_idx, S, delta, delta * rtol, all)
    if src.shape[0] == 0:
        raise ValueError(f"delta = {delta} ({associate}) produced an empty index list - "
                         "try lower values or a less strict tolerance")
    err = _errors(rt, et, r_idx[src], r_idx[tgt], e_idx[src], e_idx[tgt], S, etype)
    return _statistics(err, otype)
