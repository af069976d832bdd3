"""Model predictive control by iterative LQR (reference: pypose/module/mpc.py).  DESIGN.md §3.7."""
import torch
from torch import nn

from ..utils.stepper import ReduceToBason
from .lqr import LQR


class MPC(nn.Module):
    r"""Model predictive control: iterative LQR on the linearisation of `system` along the current inputs.

    Args:
        system: the dynamics (`LTI`, `LTV`, `NLS` or any `System`).
        Q, p, T: the cost and horizon, as for `LQR`.
        stepper: stops the iterations; default `ReduceToBason(steps=10)`.  Its step budget is reduced by one at
            construction: `steps - 1` passes run without gradients and one more, from the best of them, with gradients.

    `forward(dt, x_init, u_init=None, u_lower=None, u_upper=None, du=None)` returns (x, u, cost) of that last pass.  The
    best pass is chosen by `cost < best`, which needs a one-element cost (one problem).  Every pass takes the route of
    its `LQR`, so an `LTI` or `LTV` system runs on the CUDA kernels of csrc/lqr.cu.
    """

    def __init__(self, system, Q, p, T, stepper=None):
        super().__init__()
        self.stepper = ReduceToBason(steps=10) if stepper is None else stepper
        self.stepper.max_steps -= 1
        self.lqr = LQR(system, Q, p, T)

    def forward(self, dt, x_init, u_init=None, u_lower=None, u_upper=None, du=None):
        u, best = u_init, None
        self.stepper.reset()
        with torch.no_grad():
            while self.stepper.continual():
                x, u, cost = self.lqr(x_init, dt, u)
                self.stepper.step(cost)
                if best is None or cost < best[1]:
                    best = (u, cost)
        return self.lqr(x_init, dt, u_traj=u_init if best is None else best[0])
