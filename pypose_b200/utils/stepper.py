"""Loop steppers: objects that decide, from the loss of each pass, whether an iterative loop goes on."""
import torch


class ReduceToBason:
    """Ends a loop when the loss stops going down.

    `step(loss)` records one pass.  The loop ends (`continual()` turns False) as soon as any of these holds:

    * every loss is below `tol`;
    * `steps` passes have been recorded;
    * for `patience` passes in a row, every relative decrease `(previous - loss) / loss` was below `decreasing`.

    `loss` is a float or a tensor of any shape (a batch: each condition must hold for all of its elements).  The ratios
    and comparisons are evaluated in the loss dtype.  Before the first pass the previous loss is a float32 `inf`, so the
    first pass never counts towards the patience; a 0 / 0 ratio is NaN, compares false and resets the count.  `reset()`
    restores the initial state.  With `verbose=True` every pass and the reason for stopping are printed.

    State kept between passes: `steps`, `patience_count`, `last` (the previous loss) and `_continual`.
    `pp.module.ICP` evaluates this rule on the GPU when it is given a non-verbose `ReduceToBason` (csrc/icp_math.cuh).
    """

    def __init__(self, steps, patience=5, decreasing=1e-3, tol=1e-5, verbose=False):
        self.max_steps = steps
        self.patience = patience
        self.decreasing = decreasing
        self.tol = tol
        self.verbose = verbose
        self.reset()

    def reset(self):
        self.steps = 0
        self.patience_count = 0
        self.last = torch.tensor(float("inf"))
        self._continual = True

    def continual(self):
        return self._continual

    def _stop(self, reason):
        self._continual = False
        if self.verbose:
            print(f"ReduceToBason: stopping after step {self.steps}: {reason}")

    def step(self, loss):
        loss = loss if torch.is_tensor(loss) else torch.tensor(loss)
        if self.verbose:
            print(f"ReduceToBason: step {self.steps}, loss {loss}")
        self.steps += 1
        flat = bool(torch.all((self.last - loss) / loss < self.decreasing))
        self.patience_count = self.patience_count + 1 if flat else 0
        self.last = loss
        if bool(torch.all(loss < self.tol)):
            self._stop(f"loss below tol = {self.tol}")
        if self.steps >= self.max_steps:
            self._stop(f"reached the maximum of {self.max_steps} steps")
        if self.patience_count >= self.patience:
            self._stop(f"relative decrease below {self.decreasing} for {self.patience} steps")
