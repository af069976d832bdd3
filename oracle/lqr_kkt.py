"""fp64 dense-KKT oracle of the affine LQR problem, independent of the Riccati recursion and its adjoint.

For x' = A_t x + B_t u + c1_t the affine route of pp.module.LQR returns the stationary point of one equality-constrained
QP per problem:

    minimise   sum_t 1/2 tau_t^T Q_t tau_t + p_t^T tau_t      over tau_t = [x_t; u_t] (t < T) and x_T
    subject to x_0 = x_init,  x_{t+1} = A_t x_t + B_t u_t + c1_t.

`solve` builds the KKT matrix of that QP for every problem and solves it with one `torch.linalg.solve`; gradients are
taken by autograd through that solve.  Operands are torch tensors (nb|1, T|1, ...), broadcast here, so the gradient of a
broadcast operand comes out summed over its broadcast axes.  Q enters through its symmetric part, the only part the
problem depends on, so its gradient is symmetric.  Keep T * n to a few thousand: the solve is dense.
"""
import torch


def _full(a, nb, T, tail):
    return a.to(torch.float64).expand((nb, T) + tuple(tail))


def solve(Q, p, A, B, c1, x_init, T):
    """-> x (nb, T+1, ns), u (nb, T, nc), cost (nb) of the minimiser; c1 may be None (zeros)."""
    nb, ns = x_init.shape
    n = p.shape[-1]
    nc = n - ns
    Q, p, A, B = _full(Q, nb, T, (n, n)), _full(p, nb, T, (n,)), _full(A, nb, T, (ns, ns)), _full(B, nb, T, (ns, nc))
    c1 = x_init.new_zeros((nb, T, ns), dtype=torch.float64) if c1 is None else _full(c1, nb, T, (ns,))
    x_init = x_init.to(torch.float64)
    Qs = 0.5 * (Q + Q.mT)
    N, M = T * n + ns, (T + 1) * ns          # unknowns [tau_0, ..., tau_{T-1}, x_T]; constraints x_0, x_1, ..., x_T
    K = x_init.new_zeros((nb, N + M, N + M), dtype=torch.float64)
    rhs = x_init.new_zeros((nb, N + M), dtype=torch.float64)
    eye = torch.eye(ns, dtype=torch.float64, device=x_init.device)
    xcol = lambda t: t * n if t < T else T * n   # noqa: E731  (column of x_t)
    for t in range(T):
        K[:, t * n:(t + 1) * n, t * n:(t + 1) * n] = Qs[:, t]
        rhs[:, t * n:(t + 1) * n] = -p[:, t]
    C = x_init.new_zeros((nb, M, N), dtype=torch.float64)
    C[:, :ns, :ns] = eye
    rhs[:, N:N + ns] = x_init
    for t in range(T):
        r = (t + 1) * ns
        C[:, r:r + ns, xcol(t + 1):xcol(t + 1) + ns] = eye
        C[:, r:r + ns, t * n:t * n + ns] = -A[:, t]
        C[:, r:r + ns, t * n + ns:(t + 1) * n] = -B[:, t]
        rhs[:, N + r:N + r + ns] = c1[:, t]
    K[:, N:, :N] = C
    K[:, :N, N:] = C.mT
    z = torch.linalg.solve(K, rhs)[:, :N]
    tau = z[:, :T * n].reshape(nb, T, n)
    x = torch.cat((tau[..., :ns], z[:, None, T * n:]), 1)
    u = tau[..., ns:]
    cost = (0.5 * torch.einsum('bti,btij,btj->b', tau, Q, tau) + torch.einsum('bti,bti->b', tau, p))
    return x, u, cost


def rollout(A, B, c1, x_init, u_traj, T):
    """x_traj (nb, T, ns): the states of u_traj (zeros when None) from x_init, x_traj[:, 0] = x_init."""
    nb, ns = x_init.shape
    nc = B.shape[-1]
    A, B = _full(A, nb, T, (ns, ns)), _full(B, nb, T, (ns, nc))
    c1 = None if c1 is None else _full(c1, nb, T, (ns,))
    u = x_init.new_zeros((nb, T, nc), dtype=torch.float64) if u_traj is None else _full(u_traj, nb, T, (nc,))
    xs = [x_init.to(torch.float64)]
    for t in range(T - 1):
        x = torch.einsum('bij,bj->bi', A[:, t], xs[-1]) + torch.einsum('bij,bj->bi', B[:, t], u[:, t])
        xs.append(x if c1 is None else x + c1[:, t])
    return torch.stack(xs, 1)


def status(Q, A, B, nb, T):
    """int32 (nb): 1 where the QP has no unique minimiser, i.e. where its Hessian reduced to the inputs (x_0 = 0,
    no affine terms) is not positive definite or not finite.  The Riccati recursion meets a Quu that is not positive
    definite exactly then: Quu_t is the Schur complement of the reduced Hessian of the tail from t on."""
    ns, nc = A.shape[-1], B.shape[-1]
    n = ns + nc
    Q, A, B = _full(Q, nb, T, (n, n)), _full(A, nb, T, (ns, ns)), _full(B, nb, T, (ns, nc))
    Qs = 0.5 * (Q + Q.mT)
    X = Q.new_zeros((nb, ns, T * nc))                 # d x_t / d (u_0, ..., u_{T-1})
    R = Q.new_zeros((nb, T * nc, T * nc))
    for t in range(T):
        U = Q.new_zeros((nb, nc, T * nc))
        U[:, :, t * nc:(t + 1) * nc] = torch.eye(nc, dtype=Q.dtype)
        Z = torch.cat((X, U), 1)                     # d tau_t / d u
        R = R + Z.mT @ Qs[:, t] @ Z
        X = A[:, t] @ X + B[:, t] @ U
    bad = ~torch.isfinite(R).flatten(1).all(1)
    info = torch.linalg.cholesky_ex(torch.where(bad[:, None, None], torch.eye(T * nc, dtype=R.dtype), R)).info
    return (bad | (info != 0)).to(torch.int32)
