"""Device-decided LM trials (csrc/lmstep.cu): one C call per trial, one host read per step.

The host loop keeps the shape of optimizer.py:659-680; what moved to the device is everything inside one trial —
linearise, solve, retract, trial loss, `strategy.update`, the accept test and the parameter update.  The host owns
`param_groups` (users and schedulers edit the damping between steps): the current values travel as arguments of the
call and the updated ones come back in the 16-double state, which is the step's only device->host read.
"""
import ctypes

import torch

from .. import _C
from . import _fused
from .strategy import Adaptive, Constant, TrustRegion

ST_STATUS, ST_LOSS, ST_LAST, ST_DAMPING, ST_RADIUS, ST_DOWN, ST_REJECT, ST_CUR, ST_TRIAL, ST_PRED, ST_FAILED = range(11)
_KIND = {Constant: 0, Adaptive: 1, TrustRegion: 2}


def strategy_kind(strategy):
    """0 / 1 / 2 for exactly the three reference strategies (a subclass may override update -> host route), else None."""
    return _KIND.get(type(strategy))


def fill_ctl(ctl, strategy, pg, last, cached, reject_count, reject_limit):
    """The 14 host doubles of b200_lm_*_step's `ctl` (layout: include/b200pose.h)."""
    kind = _KIND[type(strategy)]
    ctl[0], ctl[1], ctl[2] = last, 1.0 if cached else 0.0, pg['damping']
    ctl[4], ctl[5], ctl[6] = float(reject_count), float(reject_limit), float(kind)
    if kind == 0:
        ctl[3] = 0.0
    else:
        ctl[3], ctl[7], ctl[8], ctl[9] = pg['down'], pg['high'], pg['low'], pg['up']
        ctl[12], ctl[13] = strategy.min, strategy.max
        if kind == 2:
            ctl[10], ctl[11] = strategy.down, pg['factor']


def apply_state(strategy, pg, st):
    """param_groups <- what strategy.update would have written (strategy.py:41-46, 134-151, 248-274)."""
    kind = _KIND[type(strategy)]
    if kind == 1:
        pg['damping'] = st[ST_DAMPING]
    elif kind == 2:
        pg['radius'], pg['down'], pg['damping'] = st[ST_RADIUS], st[ST_DOWN], st[ST_DAMPING]


class DeviceStep:
    """Per-problem buffers of the device-decided route: pinned host copy of the state, host `ctl`, bound entry point."""

    def __init__(self, device, dtype):
        self.device, self.dtype = device, dtype
        self.host = torch.zeros(16, dtype=torch.float64).pin_memory()
        self.host_ptr = self.host.data_ptr()
        self.ctl = (ctypes.c_double * 14)()
        self.ctl_ptr = ctypes.addressof(self.ctl)
        self.W = _fused._workspaces(device)
        self.sfx = _C.suffix(dtype)
        self.state = None
        self.comm = None
        self.seq = 0

    def next_seq(self):
        self.seq += 1
        return self.seq

    def attach_comm(self, comm, part_off=0, pt_off=0):
        self.comm, self.part_off, self.pt_off = comm, part_off, pt_off
        self.epoch0 = self.epoch1 = 0

    def new_state(self):
        """A fresh 16-double device state per step: `optimizer.loss` / `.last` are views of it, so losses a caller keeps
        from earlier steps do not change under them."""
        self.state = torch.empty(16, dtype=torch.float64, device=self.device)
        return self.state

    def read(self):
        return self.host.tolist()


def reproj_trial(ds, prob, scale, dmin, dmax, retry):
    poses = prob._poses()
    H, g, Pt = prob._buf
    _C.enqueue("b200_lm_reproj_step_" + ds.sfx, poses, poses.data_ptr(), prob.pts.data_ptr(), prob.pix.data_ptr(),
               prob.seg.data_ptr(), H.data_ptr(), g.data_ptr(), Pt.data_ptr(), ds.W[0].data_ptr(), ds.W[1].data_ptr(),
               ds.state.data_ptr(), ds.host_ptr, ds.next_seq(), ds.ctl_ptr, int(prob.robust[0]), float(prob.robust[1]), float(scale),
               float(dmin), float(dmax), 1 if retry else 0, prob.pts.shape[0], poses.shape[0])
    return ds.read()


def poseinv_trial(ds, prob, scale, dmin, dmax, retry):
    P, X = prob._rows()
    if prob._trial is None or prob._trial.shape != P.shape:
        prob._trial = torch.empty_like(P)
    _C.enqueue("b200_lm_poseinv_step_" + ds.sfx, P, P.data_ptr(), X.data_ptr(), prob._trial.data_ptr(), ds.W[0].data_ptr(),
               ds.state.data_ptr(), ds.host_ptr, ds.next_seq(), ds.ctl_ptr, int(prob.robust[0]), float(prob.robust[1]), float(scale),
               float(dmin), float(dmax), P.shape[0])
    return ds.read()


def _align(n, a=256):
    return (n + a - 1) // a * a


GATHER_BYTES = 8 << 20


def reproj_gather(ncam, world, itemsize):
    """Gather form of the sharded reprojection trial (every rank receives all partial blocks and solves every camera: one
    exchange fewer per trial) while world * ncam blocks stay small; owner form (reduce-scatter + all-gather) beyond."""
    return world * ncam * 28 * itemsize <= GATHER_BYTES


def reproj_payload(ncam, world, itemsize):
    """(part_off, pt_off, bytes) of the exchange payload of b200_lm_reproj_step_peer."""
    q = ncam if reproj_gather(ncam, world, itemsize) else (ncam + world - 1) // world
    part = _align(world * q * 28 * itemsize)          # 16-byte slots: 28 numbers per partial block, 8 per trial pose
    return 0, part, part + _align(ncam * 8 * itemsize)


def _present_mask(prob, comm):
    """(world, ncam) uint8: which rank holds rows of which camera.  One all-gather when the problem is set up; a rank sends
    no block for a camera it has no rows of and the receivers skip those slots, so with rows sorted by camera before the split
    (SURVEY.md §8e) a rank's accumulate pass only touches its own cameras."""
    import torch.distributed as dist
    mine = (prob.seg[1:] > prob.seg[:-1]).to(torch.uint8).contiguous()
    out = [torch.empty_like(mine) for _ in range(comm.world)]
    dist.all_gather(out, mine, group=None if prob.group is True else prob.group)
    return torch.stack(out).contiguous(), torch.nonzero(mine).flatten().to(torch.int32).contiguous()


def reproj_trial_peer(ds, prob, scale, dmin, dmax, retry):
    poses = prob._poses()
    H, g, _ = prob._buf
    c = ds.comm
    if getattr(ds, 'present_for', None) is not prob.seg:
        (ds.present, ds.cams), ds.present_for = _present_mask(prob, c), prob.seg
    if not retry:
        ds.epoch0 += 1
    ds.epoch1 += 1
    _C.enqueue("b200_lm_reproj_step_peer_" + ds.sfx, poses, poses.data_ptr(), prob.pts.data_ptr(), prob.pix.data_ptr(),
               prob.seg.data_ptr(), H.data_ptr(), g.data_ptr(), c.bases_ptr, c.rank, c.world, ds.part_off, ds.pt_off,
               ds.epoch0, ds.epoch1, ds.W[0].data_ptr(), ds.W[1].data_ptr(), ds.W[2].data_ptr(), ds.state.data_ptr(),
               ds.host_ptr, ds.next_seq(), ds.ctl_ptr, int(prob.robust[0]), float(prob.robust[1]), float(scale), float(dmin), float(dmax),
               1 if retry else 0, prob.pts.shape[0], 1 if reproj_gather(poses.shape[0], c.world, poses.element_size()) else 0,
               ds.present.data_ptr(), ds.cams.data_ptr(), ds.cams.shape[0], poses.shape[0])
    return ds.read()


def poseinv_trial_peer(ds, prob, scale, dmin, dmax, retry):
    P, X = prob._rows()
    if prob._trial is None or prob._trial.shape != P.shape:
        prob._trial = torch.empty_like(P)
    c = ds.comm
    ds.epoch1 += 1
    _C.enqueue("b200_lm_poseinv_step_peer_" + ds.sfx, P, P.data_ptr(), X.data_ptr(), prob._trial.data_ptr(), c.bases_ptr,
               c.rank, c.world, ds.epoch1, ds.W[0].data_ptr(), ds.state.data_ptr(), ds.host_ptr, ds.next_seq(), ds.ctl_ptr,
               int(prob.robust[0]), float(prob.robust[1]), float(scale), float(dmin), float(dmax), P.shape[0])
    return ds.read()


# ----------------------------------------------------------------------------------------------------------------
# native step driver of the block-sparse pose families (csrc/lmdrive.cu b200_lm_pgo2_step)
# ----------------------------------------------------------------------------------------------------------------
class PgoStepArgs(ctypes.Structure):
    """Mirror of `b200_pgo_step_args` (include/b200pose.h)."""
    _vp, _ip, _dp = ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p
    _fields_ = ([(n, ctypes.c_int) for n in ("family", "is64", "robust", "retry")]
                + [(n, ctypes.c_longlong) for n in ("N", "E", "maxiter", "hint", "seq", "iters_out")]
                + [(n, ctypes.c_double) for n in ("delta", "scale", "dmin", "dmax", "tol")]
                + [("intr", ctypes.c_double * 5), ("ctl", ctypes.c_double * 14)]
                + [(n, ctypes.c_void_p) for n in ("nodes", "Z", "pts", "pix", "pseg", "pa", "pb", "ei", "ej", "epos_i", "epos_j",
                                                  "nother", "nptr", "Mn", "un", "Hd", "g", "extra", "Minv", "x", "r", "z", "p0",
                                                  "p1", "q", "xbest", "X7", "Pt", "ws0", "ws1", "ws2", "ws3", "cg", "st", "host")])


class PgoDeviceStep:
    """Buffers + argument block of one pose-graph-structured problem; `trial` is one C call."""

    def __init__(self, prob, nodes):
        dev, dt = nodes.device, nodes.dtype
        N, E = nodes.shape[0], prob.ei.shape[0]
        self.device, self.dtype, self.comm = dev, dt, None
        new = lambda *shape: torch.empty(*shape, dtype=dt, device=dev)
        family = {"pgo": 0, "reproj2": 1, "sim3": 2, "so3": 3}[prob.kind]
        W = _fused.KIND_WIDTH[prob.kind]
        slot, pw, D = _fused.NODE_WIDTHS[W][:3]         # slot words, packed block words, parameter width (include/b200pose.h)
        self.buf = {"Mn": new(2 * E, slot), "un": new(2 * E, W), "Hd": new(N, pw), "g": new(N, W), "extra": new(N, W),
                    "Minv": new(N, pw), "x": new(N, W), "r": new(N, W), "z": new(N, W), "p0": torch.zeros(N, W, dtype=dt, device=dev),
                    "p1": torch.zeros(N, W, dtype=dt, device=dev), "q": new(N, W), "xbest": new(N, W), "X7": new(N, D),
                    "Pt": new(N, D)}
        n = _C.lib().b200_lm_workspace_doubles
        n.restype = ctypes.c_longlong
        self.W = torch.zeros(4, int(n()), dtype=torch.float64, device=dev)        # this problem's own reduction slots
        self.cg = torch.zeros(16, dtype=torch.float64, device=dev)
        self.host = torch.zeros(40, dtype=torch.float64).pin_memory()
        self.state = None
        a = self.args = PgoStepArgs()
        a.family, a.is64 = family, int(dt == torch.float64)
        a.N, a.E = N, E
        a.Z = prob.Z.data_ptr() if prob.Z is not None else None
        if prob.kind == "reproj2":
            a.pts, a.pix, a.pseg, a.pa, a.pb = (t.data_ptr() for t in (prob.pts, prob.pix, prob.pseg, prob.pa, prob.pb))
            for i, v in enumerate(prob.intr):
                a.intr[i] = v
        for name in ("ei", "ej", "epos_i", "epos_j", "nother", "nptr"):
            setattr(a, name, getattr(prob, name).data_ptr())
        for name, t in self.buf.items():
            setattr(a, name, t.data_ptr())
        a.ws0, a.ws1, a.ws2, a.ws3 = (self.W[i].data_ptr() for i in range(4))
        a.cg, a.host = self.cg.data_ptr(), self.host.data_ptr()
        self.ctl = a.ctl
        self.seq = 0
        self.fn = _C.lib().b200_lm_pgo2_step
        self.fn.restype, self.fn.argtypes = ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]

    def new_state(self):
        self.state = torch.empty(16, dtype=torch.float64, device=self.device)
        self.args.st = self.state.data_ptr()
        return self.state

    def trial(self, prob, nodes, scale, dmin, dmax, retry):
        a = self.args
        self.seq += 1
        a.nodes = nodes.data_ptr()
        a.robust, a.delta = int(prob.robust[0]), float(prob.robust[1])
        a.scale, a.dmin, a.dmax, a.tol = float(scale), float(dmin), float(dmax), float(prob.tol)
        a.maxiter = int(prob.maxiter) if prob.maxiter is not None else 0
        a.hint = prob.cg_iters + 1 if prob.cg_iters else 0
        a.retry, a.seq = (1 if retry else 0), self.seq
        rc = self.fn(ctypes.addressof(a), torch._C._cuda_getCurrentRawStream(self.device.index))
        if rc != 0:
            raise _C.B200PoseError(f"b200_lm_pgo2_step failed with CUDA error {rc}")
        prob.cg_iters = int(a.iters_out)
        return self.host[:16].tolist()


class BaStepArgs(ctypes.Structure):
    """Mirror of `b200_ba_step_args` (include/b200pose.h)."""
    _fields_ = ([(n, ctypes.c_int) for n in ("is64", "robust", "retry", "tpi")]
                + [(n, ctypes.c_longlong) for n in ("C", "P", "m", "split", "maxiter", "hint", "seq", "iters_out")]
                + [(n, ctypes.c_double) for n in ("delta", "scale", "dmin", "dmax", "tol")]
                + [("ctl", ctypes.c_double * 14)]
                + [(n, ctypes.c_void_p) for n in ("poses", "points", "pix", "pidx", "cidx", "cseg", "ppos", "cidx_p", "pptr", "pix_p",
                                                  "Y4", "Y4p", "rs", "Hcc", "gc", "Hpp", "gp", "part", "Hc", "Hpinv", "Minv", "Sd",
                                                  "bneg", "x", "r", "z", "p", "q", "t", "xbest", "xp", "X7", "Tn", "pn",
                                                  "ws0", "ws1", "ws2", "ws3", "cg", "st", "host")])


class BaDeviceStep:
    """Buffers + argument block of one bundle-adjustment problem; `trial` is one C call (csrc/lmdrive.cu b200_lm_ba_step)."""

    def __init__(self, prob, T, pts):
        dev, dt = T.device, T.dtype
        C, P, m = T.shape[0], pts.shape[0], prob.pix.shape[0]
        cseg, split, tpi, ppos, cidx_p, pptr, pix_p = prob.geom
        self.device, self.dtype, self.comm = dev, dt, None
        new = lambda *shape: torch.empty(*shape, dtype=dt, device=dev)
        self.buf = {"Y4": new(m, 4), "Y4p": new(m, 4), "rs": new(m, 2), "Hcc": new(C, 21), "gc": new(C, 6), "Hpp": new(P, 6),
                    "gp": new(P, 3), "part": new(max(C * split, 1), 27), "Hc": new(C, 21), "Hpinv": new(P, 6), "Minv": new(C, 21),
                    "Sd": new(C, 21), "bneg": new(C, 6), "x": new(C, 6), "r": new(C, 6), "z": new(C, 6), "p": new(C, 6),
                    "q": new(C, 6), "t": new(P, 3), "xbest": new(C, 6), "xp": new(P, 3), "X7": new(C, 7), "Tn": new(C, 7),
                    "pn": new(P, 3)}
        n = _C.lib().b200_lm_workspace_doubles
        n.restype = ctypes.c_longlong
        self.W = torch.zeros(4, int(n()), dtype=torch.float64, device=dev)
        self.cg = torch.zeros(16, dtype=torch.float64, device=dev)
        self.host = torch.zeros(40, dtype=torch.float64).pin_memory()
        self.state = None
        a = self.args = BaStepArgs()
        a.is64, a.tpi = int(dt == torch.float64), int(tpi)
        a.C, a.P, a.m, a.split = C, P, m, int(split)
        for name, t in (("pix", prob.pix), ("pidx", prob.pidx), ("cidx", prob.cidx), ("cseg", cseg), ("ppos", ppos),
                        ("cidx_p", cidx_p), ("pptr", pptr), ("pix_p", pix_p)):
            setattr(a, name, t.data_ptr())
        for name, t in self.buf.items():
            setattr(a, name, t.data_ptr())
        a.ws0, a.ws1, a.ws2, a.ws3 = (self.W[i].data_ptr() for i in range(4))
        a.cg, a.host = self.cg.data_ptr(), self.host.data_ptr()
        self.ctl = a.ctl
        self.seq = 0
        self.fn = _C.lib().b200_lm_ba_step
        self.fn.restype, self.fn.argtypes = ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]

    def new_state(self):
        self.state = torch.empty(16, dtype=torch.float64, device=self.device)
        self.args.st = self.state.data_ptr()
        return self.state

    def trial(self, prob, T, pts, scale, dmin, dmax, retry):
        a = self.args
        self.seq += 1
        a.poses, a.points = T.data_ptr(), pts.data_ptr()
        a.robust, a.delta = int(prob.robust[0]), float(prob.robust[1])
        a.scale, a.dmin, a.dmax, a.tol = float(scale), float(dmin), float(dmax), float(prob.tol)
        a.maxiter = int(prob.maxiter) if prob.maxiter is not None else 0
        a.hint = prob.cg_iters + 1 if prob.cg_iters else 0
        a.retry, a.seq = (1 if retry else 0), self.seq
        rc = self.fn(ctypes.addressof(a), torch._C._cuda_getCurrentRawStream(self.device.index))
        if rc != 0:
            raise _C.B200PoseError(f"b200_lm_ba_step failed with CUDA error {rc}")
        prob.cg_iters = int(a.iters_out)
        return self.host[:16].tolist()
