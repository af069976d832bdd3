"""Peer-memory communicator over NVLink (csrc/comm.cu, comm.cuh): one process per GPU, one exchange buffer per rank.

`torch.distributed` is used for plumbing only — shipping the 64-byte IPC handles at set-up and a barrier at tear-down.
The data path (partial block sums, scalar sums, CG vectors) is moved by the LM kernels themselves with plain stores into
the peer's buffer.  `PeerComm.create` returns None when the exchange cannot be set up (CPU tensors, gloo, a peer on
another node, IPC refused); callers then keep the torch.distributed all-reduce route.
"""
import ctypes
import os

import torch

from . import _C

_bound = False


def _bind():
    global _bound
    if _bound:
        return
    L = _C.lib()
    vp, ll, i = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int
    L.b200_comm_alloc.argtypes, L.b200_comm_alloc.restype = [ll, ctypes.POINTER(vp)], i
    L.b200_comm_free.argtypes, L.b200_comm_free.restype = [vp], i
    L.b200_comm_export.argtypes, L.b200_comm_export.restype = [vp, vp], i
    L.b200_comm_open.argtypes, L.b200_comm_open.restype = [vp, ctypes.POINTER(vp)], i
    L.b200_comm_close.argtypes, L.b200_comm_close.restype = [vp], i
    L.b200_comm_data_offset.argtypes, L.b200_comm_data_offset.restype = [], ll
    for sfx in ("f32", "f64"):
        f = getattr(L, f"b200_comm_allreduce_{sfx}")
        f.argtypes, f.restype = [vp, vp, ll, vp, i, i, ll, ll, i, ll, vp, vp], i
    _bound = True


class PeerComm:
    """Exchange buffers of all ranks of `group`, mapped into this process."""

    def __init__(self, group, device, payload_bytes):
        import torch.distributed as dist
        _bind()
        L = _C.lib()
        self.group = None if group is True else group
        self.rank, self.world = dist.get_rank(self.group), dist.get_world_size(self.group)
        if self.world > 8:
            raise _C.B200PoseError("peer exchange supports up to 8 ranks (one NVSwitch domain)")
        self.device = device
        self.data_offset = int(L.b200_comm_data_offset())
        self.bytes = self.data_offset + int(payload_bytes)
        self.local = ctypes.c_void_p()
        with torch.cuda.device(device):
            _C.check(L.b200_comm_alloc(self.bytes, ctypes.byref(self.local)), "b200_comm_alloc")
            h = (ctypes.c_char * 64)()
            _C.check(L.b200_comm_export(self.local, ctypes.cast(h, ctypes.c_void_p)), "b200_comm_export")
            mine = (bytes(h), os.uname().nodename, self.bytes)
            everyone = [None] * self.world
            dist.all_gather_object(everyone, mine, group=self.group)
            if any(e[1] != mine[1] or e[2] != mine[2] for e in everyone):
                L.b200_comm_free(self.local)
                raise _C.B200PoseError("peer exchange needs all ranks on one node with equal buffer sizes")
            self.bases = (ctypes.c_ulonglong * 8)()
            self.opened = []
            for r, (hb, _, _) in enumerate(everyone):
                if r == self.rank:
                    self.bases[r] = self.local.value
                    continue
                p = ctypes.c_void_p()
                buf = ctypes.create_string_buffer(hb, 64)
                _C.check(L.b200_comm_open(ctypes.cast(buf, ctypes.c_void_p), ctypes.byref(p)), "b200_comm_open")
                self.bases[r] = p.value
                self.opened.append(p)
        self.bases_ptr = ctypes.addressof(self.bases)
        self.tickets = torch.zeros(16, dtype=torch.int32, device=device)
        self.epochs = {}
        dist.barrier(group=self.group)

    @classmethod
    def create(cls, group, device, payload_bytes):
        """PeerComm or None (no NCCL group / not CUDA / IPC unavailable)."""
        import torch.distributed as dist
        if group is None or device.type != "cuda":
            return None
        if not (dist.is_available() and dist.is_initialized()):
            return None
        g = None if group is True else group
        if dist.get_world_size(g) < 2 or dist.get_backend(g) != "nccl":
            return None
        ok, comm = 1, None
        try:
            comm = cls(group, device, payload_bytes)
        except Exception:                     # noqa: BLE001  (every rank must learn about a failure on any rank)
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=g)
        if int(flag.item()) == 0:
            if comm is not None:
                comm.close()
            return None
        return comm

    @classmethod
    def for_allreduce(cls, group, device, max_elems, itemsize):
        """Communicator whose payload holds the staging + result areas of sum all-reduces of up to `max_elems` elements."""
        import torch.distributed as dist
        if group is None or not (dist.is_available() and dist.is_initialized()):
            return None
        world = dist.get_world_size(None if group is True else group)
        q = ((max_elems + 3) // 4 + world - 1) // world * 4
        stage = (world * q * itemsize + 255) // 256 * 256
        result = (max_elems * itemsize + 255) // 256 * 256
        comm = cls.create(group, device, stage + result)
        if comm is not None:
            comm.stage_off, comm.result_off, comm.max_elems = 0, stage, max_elems
        return comm

    def pcg_args(self):
        """(bases, rank, world, stage, result, epoch so far, tickets) for b200_lm_*_pcg."""
        return [self.bases_ptr, self.rank, self.world, self.stage_off, self.result_off, self.epochs.get(6, 0),
                self.tickets.data_ptr()]

    def consumed(self, count, channel=6):
        self.epochs[channel] = self.epochs.get(channel, 0) + int(count)

    def sum_(self, t):
        """In-place sum over ranks through the areas reserved by for_allreduce."""
        assert t.is_contiguous() and t.numel() <= self.max_elems
        return self.allreduce_(t, self.stage_off, self.result_off)

    def next_epoch(self, channel):
        e = self.epochs.get(channel, 0) + 1
        self.epochs[channel] = e
        return e

    def allreduce_(self, t, stage, result, channel=6):
        """In-place sum over ranks of a contiguous fp32 / fp64 CUDA tensor, on the current stream, no host sync.
        stage / result: byte offsets inside the payload (staging: world * ceil(n / world) elements, result: n)."""
        n = t.numel()
        sym = f"b200_comm_allreduce_{_C.suffix(t.dtype)}"
        f = getattr(_C.lib(), sym)
        rc = f(t.data_ptr(), t.data_ptr(), n, self.bases_ptr, self.rank, self.world, int(stage), int(result), int(channel),
               self.next_epoch(channel), self.tickets.data_ptr(), torch._C._cuda_getCurrentRawStream(self.device.index))
        _C.check(rc, sym)
        return t

    def close(self):
        L = _C.lib()
        if self.local is None:
            return
        try:
            torch.cuda.synchronize(self.device)
            import torch.distributed as dist
            if dist.is_initialized():
                dist.barrier(group=self.group)
        except Exception:                     # noqa: BLE001
            pass
        for p in self.opened:
            L.b200_comm_close(p)
        L.b200_comm_free(self.local)
        self.local, self.opened = None, []
