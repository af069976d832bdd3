"""GPU: the TMA shell deals its 256-row tiles round-robin to the CTAs of a persistent grid (CTA b takes tiles b, b + grid,
b + 2 grid, ..., DESIGN.md §3.1).  Row counts are chosen against that grid (fewer tiles than CTAs, exactly as many, one
more, one fewer and one more than three rounds, a short last tile, a remainder of 1 to 3 rows for the plain-load tail,
and bench.py's 1e6 rows) for a 1 -> 1, a 2 -> 1, a 2 -> 2 and a 3 -> 2 entry point in fp32 and fp64.  Each result must
equal, bit for bit, what the plain-load shell gives for the same rows (reached through views whose base is one element
past a 16-byte boundary), and must leave the guard elements behind every output alone.  One more case queues Exp -> Log
on a side stream, eagerly and in a captured CUDA graph, against the same launches with a synchronize in between."""
import ctypes

import pytest
import torch

from pypose_b200 import _C
from pypose_b200._optable import lie_symbols

pytestmark = pytest.mark.gpu

TILE = 256
GUARD = 64
SENTINEL = -777.0
OPS = ["b200_se3_exp_fwd", "b200_SE3_mul_fwd", "b200_SE3_mul_bwd", "b200_SE3_act_bwd"]
WIDTHS = {s: ([w for _, w in ins], [w for _, w in outs]) for s, _, ins, outs, _ in lie_symbols()}


def grid_of(sym, dtype):
    """CTAs of one full launch of the TMA shell: SMs x half of the CTAs whose input and output rings fit in one SM's
    shared memory (S = 3 input stages in fp32, 2 in fp64, 2 output stages, 1 KB reserved per CTA, at most 8 CTAs of 256
    threads).  If registers limited the residency further, the sizes below would only be less pointed, not wrong."""
    ins, outs = WIDTHS[f"{sym}_{_C.suffix(dtype)}"]
    stages = 3 if dtype == torch.float32 else 2
    nbytes = (stages * sum(ins) + 2 * sum(outs)) * TILE * dtype.itemsize + 8 * stages
    props = torch.cuda.get_device_properties(0)
    occ = min(8, getattr(props, "shared_memory_per_multiprocessor", 228 * 1024) // (nbytes + 1024))
    return props.multi_processor_count * max(1, occ // 2)


def sizes(grid):
    return {"half_round": (grid // 2) * TILE, "one_round": grid * TILE, "one_round_plus_tile": (grid + 1) * TILE,
            "three_rounds_minus_tile": (3 * grid - 1) * TILE, "three_rounds_plus_tile": (3 * grid + 1) * TILE,
            "short_last_tile": 2 * grid * TILE + 100, "rem1": (grid + 1) * TILE + 41, "rem2": (grid + 1) * TILE + 42,
            "rem3": (grid + 1) * TILE + 43, "bench": 1_000_000}


def guarded(n, w, dtype, lead):
    """(whole buffer, (n, w) view starting `lead` elements in); everything outside the view is SENTINEL"""
    buf = torch.full((lead + n * w + GUARD,), SENTINEL, device="cuda", dtype=dtype)
    return buf, buf[lead:lead + n * w].view(n, w)


def run(sym, ins, n, dtype, lead):
    """Launch `sym` on copies of `ins` placed `lead` elements into their buffers; returns the outputs after checking the guards."""
    _, wo = WIDTHS[f"{sym}_{_C.suffix(dtype)}"]
    moved = []
    for t in ins:
        _, v = guarded(n, t.shape[1], dtype, lead)
        v.copy_(t)
        moved.append(v)
    outs = [guarded(n, w, dtype, lead) for w in wo]
    name = f"{sym}_{_C.suffix(dtype)}"
    sp = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _C.check(_C.fn(name)(*[v.data_ptr() for v in moved], *[v.data_ptr() for _, v in outs], n, sp), name)
    torch.cuda.synchronize()
    for (buf, v), w in zip(outs, wo):
        assert (buf[:lead] == SENTINEL).all() and (buf[lead + n * w:] == SENTINEL).all(), f"{name}: guard overwritten (n={n})"
    return [v for _, v in outs]


def inputs(sym, n, dtype):
    g = torch.Generator(device="cuda").manual_seed(n % 100003 + OPS.index(sym))
    wi, _ = WIDTHS[f"{sym}_{_C.suffix(dtype)}"]
    ins = []
    for w in wi:
        t = torch.randn(n, 6 if w == 7 else w, generator=g, device="cuda", dtype=dtype) * 0.8
        ins.append(_C.launch_rows("b200_se3_exp_fwd", [t], [7])[0] if w == 7 else t)   # width 7: valid SE3 rows
    return ins


@pytest.mark.parametrize("size", list(sizes(1)))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("sym", OPS)
def test_round_robin_tiles_match_plain_load_shell(sym, dtype, size):
    n = sizes(grid_of(sym, dtype))[size]
    ins = inputs(sym, n, dtype)
    got = run(sym, ins, n, dtype, lead=0)          # torch allocations are 512 B aligned: the TMA shell
    want = run(sym, ins, n, dtype, lead=1)         # one element in: the plain-load shell
    for k, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), f"{sym} {dtype} n={n} ({size}): output {k} differs between the shells"


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("size", ["three_rounds_plus_tile", "rem3", "bench"])
def test_queued_exp_log_matches_synchronized(size, graph):
    dtype = torch.float32
    n = sizes(grid_of("b200_se3_exp_fwd", dtype))[size]
    x = inputs("b200_se3_exp_fwd", n, dtype)[0]
    f_exp, f_log = _C.fn("b200_se3_exp_fwd_f32"), _C.fn("b200_SE3_log_fwd_f32")

    def step(X, y, sync):
        sp = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _C.check(f_exp(x.data_ptr(), X.data_ptr(), n, sp), "exp")
        sync()
        _C.check(f_log(X.data_ptr(), y.data_ptr(), n, sp), "log")
        sync()

    new = lambda: (torch.zeros(n, 7, device="cuda"), torch.zeros(n, 6, device="cuda"))   # noqa: E731
    X0, y0 = new()
    step(X0, y0, torch.cuda.synchronize)
    X1, y1 = new()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            step(X1, y1, lambda: None)
        g.replay()
    else:
        with torch.cuda.stream(side):
            step(X1, y1, lambda: None)
    torch.cuda.synchronize()
    assert torch.equal(X1, X0) and torch.equal(y1, y0), f"queued Exp -> Log differs (n={n}, graph={graph})"
