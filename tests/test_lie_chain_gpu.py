"""GPU: Lie launches that depend on each other, queued back to back on one stream, give bit for bit what the same
launches give with a stream synchronize after each one.  Back to back, the CTAs of the next launch of the TMA shell
are resident beside the running one (programmatic dependent launch, DESIGN.md §3.1) and must still read only what
the previous launch has finished writing."""
import pytest
import torch

from pypose_b200 import _C

pytestmark = pytest.mark.gpu


def exp_log_exp(x, sync):
    X = _C.launch_rows("b200_se3_exp_fwd", [x], [7])[0]
    sync()
    y = _C.launch_rows("b200_SE3_log_fwd", [X], [6])[0]
    sync()
    Z = _C.launch_rows("b200_se3_exp_fwd", [y], [7])[0]
    sync()
    return X, y, Z


# 2e6 rows: every CTA of the shell runs many tiles; 300001 rows: n % 4 != 0, so each op ends with the tail launch
@pytest.mark.parametrize("n", [2_000_000, 300_001])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_chained_launches_match_synchronized(n, dtype):
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, 6, generator=g, device="cuda", dtype=dtype) * 0.8
    chained = exp_log_exp(x, lambda: None)
    synced = exp_log_exp(x, torch.cuda.synchronize)
    for name, a, b in zip(("Exp", "Log", "Exp"), chained, synced):
        assert torch.equal(a, b), f"{name} differs when chained (n={n}, {dtype})"
