"""GPU: Lie launches queued back to back on a stream of their own, eagerly and inside one captured CUDA graph, give bit
for bit what the same launches give with a synchronize after each one.  Queued, the CTAs of the next launch of the TMA
shell are resident beside the running one (programmatic dependent launch, DESIGN.md §3.1), and each launch releases
the next only once its own predecessor has completed.  The cases cover every way one launch can depend on earlier
ones: reading what the previous launch writes through its first or its second input, writing what the previous launch
reads, in place, reading what a long launch wrote behind a tiny unrelated one, and reading what a torch kernel between
two Lie launches wrote; plus bench.py's step, where each launch reads what an earlier one wrote."""
import ctypes

import pytest
import torch

from pypose_b200 import _C

pytestmark = pytest.mark.gpu

OPS = {"exp": "b200_se3_exp_fwd", "log": "b200_SE3_log_fwd", "inv": "b200_SE3_inv_fwd", "mul": "b200_SE3_mul_fwd"}


def launcher(sync):
    def launch(op, ins, outs):
        sym = f"{OPS[op]}_{_C.suffix(ins[0].dtype)}"
        sp = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _C.check(_C.fn(sym)(*[t.data_ptr() for t in ins + outs], ins[0].shape[0], sp), sym)
        sync()
    return launch


def buffers(n, dtype):
    """Seeded inputs and outputs of one run: se3 rows a, c; SE3 rows B, B2; outputs A, C, D, b."""
    g = torch.Generator(device="cuda").manual_seed(n + (dtype == torch.float64))
    se3 = lambda m: torch.randn(m, 6, generator=g, device="cuda", dtype=dtype) * 0.8   # noqa: E731
    SE3 = lambda m: _C.launch_rows("b200_se3_exp_fwd", [se3(m)], [7])[0]              # noqa: E731
    t = {"a": se3(n), "c": se3(n), "B": SE3(n), "B2": SE3(n)}
    t.update({k: torch.zeros(n, w, device="cuda", dtype=dtype) for k, w in (("A", 7), ("C", 7), ("D", 7), ("b", 6))})
    torch.cuda.synchronize()
    return t


def independent(t, L, sync):
    """bench.py's step: each launch reads what an earlier launch, not the previous one, wrote"""
    L("exp", [t["a"]], [t["A"]])
    L("log", [t["B"]], [t["b"]])
    L("exp", [t["c"]], [t["C"]])
    return "A", "b", "C"


def first_input(t, L, sync):
    """Log reads what Exp writes"""
    L("exp", [t["a"]], [t["A"]])
    L("log", [t["A"]], [t["b"]])
    return "A", "b"


def second_input(t, L, sync):
    """Mul's first input is independent, its second is what Exp writes"""
    L("exp", [t["a"]], [t["A"]])
    L("mul", [t["B"], t["A"]], [t["D"]])
    return "A", "D"


def write_after_read(t, L, sync):
    """Exp overwrites the buffer Log reads"""
    L("log", [t["B"]], [t["b"]])
    L("exp", [t["c"]], [t["B"]])
    return "b", "B"


def in_place(t, L, sync):
    """Inv in place on a buffer the previous launch does not write, then on the one it does, then Log of the first"""
    L("exp", [t["a"]], [t["A"]])
    L("inv", [t["B"]], [t["B"]])
    L("inv", [t["A"]], [t["A"]])
    L("log", [t["B"]], [t["b"]])
    return "A", "B", "b"


def behind_tiny_launch(t, L, sync):
    """Log reads what the long Exp two launches back writes; the 4-row Exp in between shares nothing with either"""
    L("exp", [t["a"]], [t["A"]])
    L("exp", [t["c"][:4]], [t["C"][:4]])
    L("log", [t["A"]], [t["b"]])
    return "A", "C", "b"


def behind_torch_kernel(t, L, sync):
    """a torch copy writes Log's input between two Lie launches"""
    L("exp", [t["a"]], [t["A"]])
    t["B"].copy_(t["B2"])
    sync()
    L("log", [t["B"]], [t["b"]])
    return "A", "B", "b"


CASES = [independent, first_input, second_input, write_after_read, in_place, behind_tiny_launch, behind_torch_kernel]
NOSYNC = lambda: None   # noqa: E731


# 2e6 rows: every CTA of the shell runs many tiles; 300001 rows: n % 4 != 0, so each op ends with the tail launch
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("n", [2_000_000, 300_001])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", CASES, ids=[c.__name__ for c in CASES])
def test_queued_launches_match_synchronized(case, dtype, n, graph):
    ref = buffers(n, dtype)
    names = case(ref, launcher(torch.cuda.synchronize), torch.cuda.synchronize)
    got = buffers(n, dtype)
    side = torch.cuda.Stream()
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            case(got, launcher(NOSYNC), NOSYNC)
        g.replay()
    else:
        with torch.cuda.stream(side):
            case(got, launcher(NOSYNC), NOSYNC)
    torch.cuda.synchronize()
    for k in names:
        assert torch.equal(got[k], ref[k]), f"{case.__name__}: {k} differs queued (n={n}, {dtype}, graph={graph})"
