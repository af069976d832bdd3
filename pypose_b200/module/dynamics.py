"""Dynamics models (reference: pypose/module/dynamics.py): the `System` base, linear time-invariant / time-varying
systems, non-linear systems linearised by autograd, and the `toBTN` / `runsys` helpers.  Host-side torch modules; they
are the input of `LQR` and `MPC` (module/lqr.py, DESIGN.md §3.7)."""
import torch
from torch import nn
from torch.autograd.functional import jacobian

from ..function.linalg import bmv


class System(nn.Module):
    """Base class of a discrete-time dynamical system.

    Subclasses define `state_transition(state, input, t=None)` and `observation(state, input, t=None)`.  Calling the
    module advances the system by one step and returns `(next_state, observation)`; a forward hook then increments the
    system time `_t` (an int64 buffer, read and written through `systime`)."""

    def __init__(self):
        super().__init__()
        self.register_buffer('_t', torch.tensor(0, dtype=torch.int64))
        self.register_forward_hook(self.forward_hook)

    def forward_hook(self, module, inputs, outputs):
        """Advances the system time by one step after every call."""
        self._t.add_(1)

    def reset(self, t=0):
        self._t.fill_(t)
        return self

    def forward(self, state, input):
        self.state, self.input = torch.atleast_1d(state), torch.atleast_1d(input)
        return self.state_transition(self.state, self.input), self.observation(self.state, self.input)

    def state_transition(self, state, input, t=None):
        raise NotImplementedError("The users need to define their own state transition method")

    def observation(self, state, input, t=None):
        raise NotImplementedError("The users need to define their own observation method")

    def set_refpoint(self, state=None, input=None, t=None):
        """Sets the reference point of the linearisation; a no-op for systems that are linear already."""
        return self

    @property
    def systime(self):
        """System time, advanced by one on every call."""
        return self._t

    @systime.setter
    def systime(self, t):
        self._t.copy_(t if isinstance(t, torch.Tensor) else torch.tensor(t))


class LTI(System):
    """Discrete-time linear time-invariant system

        x_{k+1} = A x_k + B u_k + c1,    y_k = C x_k + D u_k + c2

    with state and input as row vectors (the last dimension).  `A, B, C, D, c1, c2` are buffers, single or batched;
    `c1` and `c2` may be None."""

    def __init__(self, A, B, C, D, c1=None, c2=None):
        super().__init__()
        for name, value in (('_A', A), ('_B', B), ('_C', C), ('_D', D), ('_c1', c1), ('_c2', c2)):
            self.register_buffer(name, value)

    def forward(self, state, input):
        return super().forward(state, input)

    def state_transition(self, state, input):
        z = bmv(self.A, state.clone()) + bmv(self.B, input)
        return z if self.c1 is None else z + self.c1

    def observation(self, state, input):
        y = bmv(self.C, state) + bmv(self.D, input)
        return y if self.c2 is None else y + self.c2

    @property
    def A(self):
        """State matrix."""
        return self._A

    @property
    def B(self):
        """Input matrix."""
        return self._B

    @property
    def C(self):
        """Output matrix."""
        return self._C

    @property
    def D(self):
        """Feed-through (observation) matrix."""
        return self._D

    @property
    def c1(self):
        """Constant term of the state transition."""
        return self._c1

    @property
    def c2(self):
        """Constant term of the observation."""
        return self._c2


class LTV(LTI):
    """Discrete-time linear time-varying system: an `LTI` whose matrices depend on the system time.  Subclasses override
    the `A, B, C, D, c1, c2` properties as functions of `_t`; `set_refpoint(t=...)` sets the system time."""

    def __init__(self, A=None, B=None, C=None, D=None, c1=None, c2=None):
        super().__init__(A, B, C, D, c1, c2)

    def set_refpoint(self, state=None, input=None, t=None):
        self.systime = t
        return self


class NLS(System):
    """Discrete-time non-linear system x_{k+1} = f(x_k, u_k, t_k), y_k = g(x_k, u_k, t_k).

    Subclasses define `state_transition(state, input, t)` (f) and `observation(state, input, t)` (g).  After
    `set_refpoint(state, input, t)` the properties `A, B, C, D` are the Jacobians of f and g at that point (reverse-mode,
    vectorised `torch.autograd.functional.jacobian`) and `c1 = f* - A x* - B u*`, `c2 = g* - C x* - D u*`, so that the
    linearisation is written in full states, like an `LTI`."""

    def __init__(self):
        super().__init__()
        self.jacargs = {'vectorize': True, 'strategy': 'reverse-mode'}

    def forward(self, state, input):
        self.state, self.input = torch.atleast_1d(state), torch.atleast_1d(input)
        return (self.state_transition(self.state, self.input, self.systime),
                self.observation(self.state, self.input, self.systime))

    def set_refpoint(self, state=None, input=None, t=None):
        """Linearise at (state, input, t); None takes the most recent state, input or system time."""
        self._ref_state = self.state if state is None else torch.atleast_1d(state)
        self._ref_input = self.input if input is None else torch.atleast_1d(input)
        self._ref_t = self.systime if t is None else torch.atleast_1d(t)
        self._ref_f = self.state_transition(self._ref_state, self._ref_input, self._ref_t)
        self._ref_g = self.observation(self._ref_state, self._ref_input, self._ref_t)
        return self

    def _jac(self, fn, wrt_state):
        x, u, t = self._ref_state, self._ref_input, self._ref_t
        if wrt_state:
            return jacobian(lambda s: fn(s, u, t), x, **self.jacargs)
        return jacobian(lambda i: fn(x, i, t), u, **self.jacargs)

    @property
    def A(self):
        """df/dx at the reference point."""
        return self._jac(self.state_transition, True)

    @property
    def B(self):
        """df/du at the reference point."""
        return self._jac(self.state_transition, False)

    @property
    def C(self):
        """dg/dx at the reference point."""
        return self._jac(self.observation, True)

    @property
    def D(self):
        """dg/du at the reference point."""
        return self._jac(self.observation, False)

    @property
    def c1(self):
        """f(x*, u*, t*) - A x* - B u*."""
        return self._ref_f - bmv(self.A, self._ref_state) - bmv(self.B, self._ref_input)

    @property
    def c2(self):
        """g(x*, u*, t*) - C x* - D u*."""
        return self._ref_g - bmv(self.C, self._ref_state) - bmv(self.D, self._ref_input)


def toBTN(vec, T):
    """Reshape `(..., N)` to `(B, T, N)`: 1-D and 2-D inputs gain leading axes, and a time axis of size 1 is repeated
    T times."""
    while vec.ndim < 3:
        vec = vec.unsqueeze(0)
    if vec.shape[1] == 1:
        vec = vec.repeat(1, T, 1)
    return vec


def runsys(system, T, x_traj, u_traj):
    """Roll `system` out over T steps in place of `x_traj[..., 1:, :]`, from `x_traj[..., 0, :]` and `u_traj`;
    returns the `(B, T, N)` state trajectory."""
    x_traj, u_traj = toBTN(x_traj, T), toBTN(u_traj, T)
    for i in range(T - 1):
        x_traj[..., i + 1, :], _ = system(x_traj[..., i, :], u_traj[..., i, :])
    return x_traj
