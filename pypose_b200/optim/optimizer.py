"""Gauss-Newton and Levenberg-Marquardt (reference: pypose/optim/optimizer.py).

`step()` keeps the reference's control flow and state (`loss`, `last`, `reject_count`,
`param_groups[...]['damping']`, defaults min=1e-6 / max=1e32 / reject=16, cumulative damping across
rejected trials, diagonal clamp before damping, loss cached between steps — optimizer.py:459-680).

Two routes produce the step:

* generic  — any `nn.Module`: `modjac` through the b200pose ops' backward kernels, dense J, dense
  solver objects.  Same arithmetic as the reference, O(N^2) memory; kept so nothing that ran stops running.
* structured — models whose residual family is known (optim/structured.py): one fused kernel per
  LM trial, no Jacobian in memory.  Chosen automatically when the reference's dense step would compute
  exactly the same block system (single SE3 parameter, default Cholesky solver, no kernel / weight).
"""
import torch
from torch import nn
from torch.optim import Optimizer

from .corrector import FastTriggs
from .functional import modjac
from .solver import PINV, Cholesky
from .strategy import TrustRegion
from . import _lmstep, structured


class Trivial(torch.nn.Module):
    """Identity kernel / corrector (optimizer.py:52-61)."""

    def __init__(self, *args, **kwargs):
        super().__init__()

    def forward(self, *args, **kwargs):
        out = *args, *kwargs.values()
        return out[0] if len(out) == 1 else out


class RobustModel(nn.Module):
    """Residual / loss plumbing around the user model (optimizer.py:64-125)."""

    def __init__(self, model, kernel=None, auto=False):
        super().__init__()
        self.model = model
        self.kernel = [Trivial()] if kernel is None else kernel

    def flatten_row_jacobian(self, J, params_values):
        if isinstance(J, (tuple, list)):
            J = torch.cat([j.reshape(-1, p.numel()) for j, p in zip(J, params_values)], 1)
        return J

    def normalize_RWJ(self, R, weight, J):
        weight_diag = None
        if weight is not None:
            weight = weight if isinstance(weight, (tuple, list)) else [weight]
            assert len(R) == len(weight)
            blocks = []
            for w, r in zip(weight, R):
                ni = r.numel() * w.shape[-1] / w.numel()
                w = w.view(*w.shape, 1, 1) if r.shape[-1] == 1 else w
                blocks += list(w.reshape(-1, w.shape[-2], w.shape[-1]).unbind(0)) * int(ni)
            weight_diag = torch.block_diag(*blocks)
        R = [r.reshape(-1) for r in R]
        J = torch.cat(J) if isinstance(J, (tuple, list)) else J
        return torch.cat(R), weight_diag, J

    def forward(self, input, target=None):
        return self.residuals(self.model_forward(input), target)

    def model_forward(self, input):
        if isinstance(input, dict):
            return self.model(**input)
        if isinstance(input, (tuple, list)):
            return self.model(*input)
        return self.model(input)

    def residual(self, output, target):
        return output if target is None else output - target

    def residuals(self, outputs, targets):
        if isinstance(outputs, (tuple, list)):
            targets = [None] * len(outputs) if targets is None else targets
            return tuple(self.residual(o, targets[i]) for i, o in enumerate(outputs))
        return tuple([self.residual(outputs, targets)])

    def loss(self, input, target):
        residuals = self.residuals(self.model_forward(input), target)
        kernels = self.kernel if len(self.kernel) > 1 else [self.kernel[0]] * len(residuals)
        return sum(k(r.square().sum(-1)).sum() for k, r in zip(kernels, residuals))


class _Optimizer(Optimizer):
    """Base class (optimizer.py:128-140)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)

    def update_parameter(self, params, step):
        """p.add_(d): plain addition for Tensors, left retraction Exp(d) * p for group LieTensors."""
        steps = step.split([p.numel() for p in params if p.requires_grad])
        [p.add_(d.view(p.shape)) for p, d in zip(params, steps) if p.requires_grad]


def _as_list(x):
    return list(x) if isinstance(x, (tuple, list)) else [x]


def _setup_correctors(kernel, corrector):
    if kernel is not None:
        kernel = [k if k is not None else Trivial() for k in _as_list(kernel)]
        corrector = [FastTriggs(k) for k in kernel] if corrector is None else corrector
    else:
        corrector = [Trivial()] if corrector is None else corrector
    corrector = [c if c is not None else Trivial() for c in _as_list(corrector)]
    return kernel, corrector


class _SecondOrder(_Optimizer):
    def _linearize(self, input, target, weight):
        """R (M,), W (block-diag or None), J (M, P) — optimizer.py:645-653."""
        weight = self.weight if weight is None else weight
        R = list(self.model(input, target))
        J = modjac(self.model, input=(input, target), flatten=False, **self.jackwargs)
        params_values = tuple(dict(self.model.named_parameters()).values())
        J = [self.model.flatten_row_jacobian(Jr, params_values) for Jr in J]
        for i in range(len(R)):
            c = self.corrector[0] if len(self.corrector) == 1 else self.corrector[i]
            R[i], J[i] = c(R=R[i], J=J[i])
        return self.model.normalize_RWJ(R, weight, J)


class GaussNewton(_SecondOrder):
    """Gauss-Newton (optimizer.py:143-328): D = solver(W J, -W R), default solver PINV.

    With the default solver, no kernel / weight / target and a model of a block-diagonal family (PoseInv, single-pose
    reprojection; optim/structured.py) the step is the fused LM trial without damping: the normal equations of a
    full-rank J have the pseudo-inverse's solution, so the batched 6x6 Cholesky solve replaces the dense `pinv`."""

    def __init__(self, model, solver=None, kernel=None, corrector=None, weight=None, vectorize=True, group=None):
        super().__init__(model.parameters(), defaults={})
        self.jackwargs = {'vectorize': vectorize}
        self._default_solver = solver is None
        self.solver = PINV() if solver is None else solver
        self.weight, self.group = weight, group
        self._plain = kernel is None and corrector is None
        kernel, self.corrector = _setup_correctors(kernel, corrector)
        self.model = RobustModel(model, kernel)
        self._problem = None

    def _structured(self, input, target, weight):
        if not (self._default_solver and self._plain and target is None and weight is None and self.weight is None
                and len(self.param_groups) == 1):
            return None
        if self._problem is not None and self._problem.matches(self.model.model, input):
            return self._problem
        prob = structured.recognize(self.model.model, input, self.param_groups[0]['params'], self.group, (0, 1.0), None, False)
        # only the families whose step is an exact batched 6x6 solve (the PCG families need a tolerance)
        self._problem = prob if isinstance(prob, (structured.PoseInvProblem, structured.ReprojProblem)) else None
        return self._problem

    @torch.no_grad()
    def step(self, input, target=None, weight=None):
        for pg in self.param_groups:
            prob = self._structured(input, target, weight)
            if prob is not None:
                r = prob.trial(prob.linearize(), 1.0, 1e-30, 1e38)       # no damping; clamp is a no-op on a PSD diagonal
                if r["failed"] == 0:
                    self.last = self.loss if hasattr(self, 'loss') else r["cur_t"]
                    prob.accept()
                    self.loss = r["loss_t"]
                    continue
                self._problem = None                                      # rank-deficient block: let PINV handle it
            R, weight, J = self._linearize(input, target, weight)
            A, b = (J, -R) if weight is None else (weight @ J, -weight @ R)
            D = self.solver(A=A, b=b.view(-1, 1))
            self.last = self.loss if hasattr(self, 'loss') else self.model.loss(input, target)
            self.update_parameter(params=pg['params'], step=D)
            self.loss = self.model.loss(input, target)
        return self.loss


class LevenbergMarquardt(_SecondOrder):
    """Levenberg-Marquardt (optimizer.py:331-680).

    `sparse=True` and `pp.Parameter(..., sjac=True)` (the reference's optional `bae` backend) are accepted
    and select the structured route as well.  `group` (extension): a torch.distributed process group
    over which residual-sharded block systems and the scalar loss / predicted-reduction sums are
    all-reduced, so every rank takes the same accept/reject decision.
    """

    def __init__(self, model, solver=None, strategy=None, kernel=None, corrector=None, weight=None, reject=16,
                 min=1e-6, max=1e32, vectorize=True, sparse=False, group=None):
        assert min > 0, ValueError("min value has to be positive: {}".format(min))
        assert max > 0, ValueError("max value has to be positive: {}".format(max))
        self.strategy = TrustRegion() if strategy is None else strategy
        defaults = {**{'min': min, 'max': max}, **self.strategy.defaults}
        super().__init__(model.parameters(), defaults=defaults)
        self.sparse, self.group = sparse, group
        self.jackwargs = {'vectorize': vectorize}
        self._default_solver = solver is None
        self.solver = Cholesky() if solver is None else solver
        self.reject, self.reject_count = reject, 0
        self.weight = weight
        # structured route: no kernel, or ONE known robust kernel with the default FastTriggs corrector
        self._robust = None
        if kernel is None and corrector is None:
            self._robust = (0, 1.0)
        elif corrector is None and not isinstance(kernel, (tuple, list)) and hasattr(kernel, 'b200_kind'):
            self._robust = (int(kernel.b200_kind), float(kernel.b200_delta))
        kernel, self.corrector = _setup_correctors(kernel, corrector)
        self.model = RobustModel(model, kernel)
        self._problem = None

    def update_parameter(self, params, step):
        super().update_parameter(params, step)

    # -- structured route ------------------------------------------------------------------------------
    def _structured(self, input, target, weight):
        weight = self.weight if weight is None else weight
        if not (self._robust is not None and target is None):
            return None
        from .solver import CG
        if not (isinstance(self.solver, CG) or (isinstance(self.solver, Cholesky) and not self.solver.upper)):
            return None
        if len(self.param_groups) != 1:
            return None
        if self._problem is not None and self._problem.matches(self.model.model, input, weight):
            return self._problem
        params = self.param_groups[0]['params']
        self._problem = structured.recognize(self.model.model, input, params, self.group,
                                             self._robust, self.solver, self.sparse, weight)
        if self._problem is None and weight is None and (self.sparse or isinstance(self.solver, CG)):
            # an SO3 pose graph (rotation averaging) takes its node-ordered route
            self._problem = structured.recognize_so3_graph(self.model.model, input, params, self.group, self._robust,
                                                           self.solver, self.sparse, weight)
        if self._problem is None and weight is None and (self.sparse or isinstance(self.solver, CG)):
            # not one of the fused families: per-residual Jacobian blocks for any batch-separable model of `sjac`
            # parameters (what the reference delegates to `bae`, optimizer.py:629-643)
            from . import blocks
            kernel = self.model.kernel[0] if self._robust[0] != 0 else None
            self._problem = blocks.BlockProblem.build(self.model.model, input, [p for p in params if p.requires_grad],
                                                      structured._input_key(input), self.group, kernel, self.solver,
                                                      self.model)
        return self._problem

    def _device_step(self, prob):
        """The device-decided route (optim/_lmstep.py, csrc/lmstep.cu) applies to a block-diagonal family on one GPU with
        one of the three reference strategies; everything else keeps the host-decided loop below."""
        ds = getattr(prob, 'device_step', None)
        if ds is None:
            return None
        return ds(self.strategy)

    def _step_on_device(self, prob, pg, ds):
        """optimizer.py:659-680 with the whole trial — incl. strategy.update, the accept test and the parameter update —
        on the device: one C call and ONE host read per trial; a productive step is a single trial."""
        cached = hasattr(self, 'loss')
        last_f = 0.0
        if cached:
            if getattr(self, '_loss_t', None) is not self.loss:      # loss was set / replaced from outside
                self._loss_f = float(self.loss)
            last_f = self._loss_f
        self.reject_count = 0
        scale, retry = 1.0, False
        state = ds.new_state()
        while True:
            scale *= 1.0 + pg['damping']
            _lmstep.fill_ctl(ds.ctl, self.strategy, pg, last_f, cached, self.reject_count, self.reject)
            st = prob.device_trial(ds, scale, pg['min'], pg['max'], retry)
            status = st[_lmstep.ST_STATUS]
            if not cached:                 # `self.last = self.loss = model.loss(...)` of the first ever step
                last_f, cached = st[_lmstep.ST_CUR], True
            self.last = state[_lmstep.ST_LAST]
            if status == 2.0:              # solver.py:214-215 -> optimizer.py:669-671
                print('Cholesky decomposition failed. Check your matrix (may not be positive-definite)',
                      '\nLinear solver failed. Breaking optimization step...')
                break
            _lmstep.apply_state(self.strategy, pg, st)
            self.reject_count = int(st[_lmstep.ST_REJECT])
            if status == 1.0:
                break
            retry = True                   # rejected: parameters untouched, damping already updated
        self.loss = state[_lmstep.ST_LOSS]
        self._loss_f, self._loss_t = st[_lmstep.ST_LOSS], self.loss
        return self.loss

    def _step_structured(self, prob, pg):
        """Same control flow as the dense branch below (optimizer.py:659-680), driven by host floats that
        come back from the device in ONE read per trial."""
        ds = self._device_step(prob)
        if ds is not None:
            return self._step_on_device(prob, pg, ds)
        cached = hasattr(self, 'loss')
        if cached:
            if getattr(self, '_loss_t', None) is not self.loss:      # loss was set / replaced from outside
                self._loss_f = float(self.loss)
            last_f = loss_f = self._loss_f
            self.last = self.loss
        self.reject_count = 0
        scale = 1.0                       # cumulative diagonal multiplier: A_ii <- A_ii (1 + damping) per trial
        lin = prob.linearize()
        first = True
        while first or last_f <= loss_f:
            scale *= 1.0 + pg['damping']
            r = prob.trial(lin, scale, pg['min'], pg['max'])
            if first and not cached:      # `self.last = self.loss = model.loss(...)` of the first ever step
                last_f = loss_f = r["cur"]
                self.last = self.loss = r["cur_t"]
            first = False
            if r["failed"] > 0:           # solver.py:214-215 -> optimizer.py:669-671
                print('Cholesky decomposition failed. Check your matrix (may not be positive-definite)',
                      '\nLinear solver failed. Breaking optimization step...')
                break
            loss_f, self.loss = r["loss"], r["loss_t"]
            self.strategy.update(pg, last=last_f, loss=loss_f, J=None, D=None, R=None, predicted=r["predicted"])
            if last_f < loss_f and self.reject_count < self.reject:
                loss_f, self.loss = last_f, self.last                # rejected: parameters untouched
                self.reject_count += 1
            else:
                prob.accept()
                break
        self._loss_f, self._loss_t = loss_f, self.loss
        return self.loss

    def step(self, input, target=None, weight=None):
        """One LM step.  The structured routes never build an autograd graph (their kernels are called through the C-ABI),
        so the fast path skips `torch.no_grad()` and torch.optim's profiling wrapper (`step.hooked` below): both together
        cost ~15 us of Python per step, a third of a 1e6-residual step."""
        if len(self.param_groups) == 1:
            prob = self._structured(input, target, weight)
            if prob is not None:
                ds = self._device_step(prob)
                if ds is not None:
                    return self._step_on_device(prob, self.param_groups[0], ds)
        with torch.no_grad():
            return self._step_generic(input, target, weight)

    step.hooked = True      # torch.optim.Optimizer._patch_step_function leaves an already "hooked" step alone

    # -- reference (dense) route -----------------------------------------------------------------------
    def _step_generic(self, input, target=None, weight=None):
        for pg in self.param_groups:
            prob = self._structured(input, target, weight)
            if prob is not None:
                self._step_structured(prob, pg)
                continue
            R, weight, J = self._linearize(input, target, weight)
            J_T = J.T @ weight if weight is not None else J.T
            A = J_T @ J
            A.diagonal().clamp_(pg['min'], pg['max'])
            self.last = self.loss = self.loss if hasattr(self, 'loss') else self.model.loss(input, target)
            self.reject_count = 0
            while self.last <= self.loss:
                A.diagonal().add_(A.diagonal() * pg['damping'])
                try:
                    D = self.solver(A=A, b=-J_T @ R.view(-1, 1))
                except Exception as e:
                    print(e, "\nLinear solver failed. Breaking optimization step...")
                    break
                self.update_parameter(pg['params'], D)
                self.loss = self.model.loss(input, target)
                self.strategy.update(pg, last=self.last, loss=self.loss, J=J, D=D, R=R.view(-1, 1))
                if self.last < self.loss and self.reject_count < self.reject:     # reject step
                    self.update_parameter(params=pg['params'], step=-D)
                    self.loss, self.reject_count = self.last, self.reject_count + 1
                else:
                    break
        return self.loss
