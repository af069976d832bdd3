"""fp64 numpy restatement of the affine LQR route (csrc/lqr.cu, DESIGN.md §3.7): the forward solve of pp.module.LQR for
x' = A_t x + B_t u + c1_t, and its KKT adjoint (Amos et al. 2018, "Differentiable MPC", module 1).

Every operand is given at full size: Q (nb,T,n,n), p (nb,T,n), A (nb,T,ns,ns), B (nb,T,ns,nc), c1 (nb,T,ns),
x_init (nb,ns), u_traj (nb,T,nc); `full()` broadcasts compact operands to that.
"""
import numpy as np


def full(Q, p, A, B, c1, x_init, u_traj):
    """Broadcast (nb|1, T|1, ...) operands to (nb, T, ...); c1 / u_traj may be None (zeros)."""
    nb, ns = x_init.shape
    T, n = max(Q.shape[1], p.shape[1]), p.shape[-1]
    nc = n - ns
    if u_traj is None:
        u_traj = np.zeros((nb, T, nc))
    if c1 is None:
        c1 = np.zeros((1, 1, ns))
    if u_traj.shape[1] > T:
        T = u_traj.shape[1]
    b = lambda a, tail: np.broadcast_to(np.asarray(a, np.float64), (nb, T) + tail)   # noqa: E731
    return (b(Q, (n, n)), b(p, (n,)), b(A, (ns, ns)), b(B, (ns, nc)), b(c1, (ns,)), np.asarray(x_init, np.float64),
            b(u_traj, (nc,)))


def _riccati(Q, A, B, ns):
    """K_t (T,nc,ns) of one problem and whether every Quu was positive definite; the linear terms are solved by
    `_gains` with the factors kept here."""
    T = Q.shape[0]
    Ls, Qts, ok = [], [None] * T, True
    V = None
    for t in range(T - 1, -1, -1):
        Qt = Q[t].copy()
        if t < T - 1:
            F = np.concatenate([A[t], B[t]], -1)
            Qt = Qt + (F.T @ V) @ F
        Qxx, Qxu, Qux, Quu = Qt[:ns, :ns], Qt[:ns, ns:], Qt[ns:, :ns], Qt[ns:, ns:]
        try:
            L = np.linalg.cholesky(Quu)
        except np.linalg.LinAlgError:
            return None, None, False
        K = -_cho_solve(L, Qux)
        Qts[t] = (Qt, K, L)
        V = Qxx + Qxu @ K + K.T @ Qux + (K.T @ Quu) @ K
    return Qts, V, ok


def _cho_solve(L, b):
    y = np.linalg.solve(L, b)
    return np.linalg.solve(L.T, y)


def _gains(Qts, q_of, A, B, ns, vT=None):
    """k_t of the backward recursion with linear terms q_of(t) (n,); vT (ns,) is a terminal linear term on x_T."""
    T = len(Qts)
    ks = [None] * T
    v = vT
    for t in range(T - 1, -1, -1):
        Qt, K, L = Qts[t]
        qt = q_of(t)
        if v is not None:
            qt = qt + np.concatenate([A[t], B[t]], -1).T @ v
        Qxu, Quu = Qt[:ns, ns:], Qt[ns:, ns:]
        qx, qu = qt[:ns], qt[ns:]
        k = -_cho_solve(L, qu)
        ks[t] = k
        v = qx + Qxu @ k + K.T @ qu + (K.T @ Quu) @ k
    return ks


def lqr(Q, p, A, B, c1, x_init, u_traj):
    """Full-size fp64 operands -> x (nb,T+1,ns), u (nb,T,nc), cost (nb), x_traj (nb,T,ns), status (nb) int32
    (1 where a Quu was not positive definite; that problem's outputs are NaN)."""
    nb, T, n = p.shape
    ns = x_init.shape[-1]
    nc = n - ns
    x, u = np.full((nb, T + 1, ns), np.nan), np.full((nb, T, nc), np.nan)
    cost, xtr, st = np.full(nb, np.nan), np.zeros((nb, T, ns)), np.zeros(nb, np.int32)
    for b in range(nb):
        xtr[b, 0] = x_init[b]
        for t in range(T - 1):
            xtr[b, t + 1] = A[b, t] @ xtr[b, t] + B[b, t] @ u_traj[b, t] + c1[b, t]
        Qts, _, ok = _riccati(Q[b], A[b], B[b], ns)
        if not ok:
            st[b] = 1
            continue
        tau = np.concatenate([xtr[b], u_traj[b]], -1)
        pbar = np.einsum('tij,tj->ti', Q[b], tau) + p[b]
        ks = _gains(Qts, lambda t: pbar[t], A[b], B[b], ns)
        xt, c = x_init[b].copy(), 0.0
        x[b, 0] = xt
        for t in range(T):
            K = Qts[t][1]
            ut = K @ (xt - xtr[b, t]) + ks[t] + u_traj[b, t]
            tau_t = np.concatenate([xt, ut])
            c += 0.5 * tau_t @ Q[b, t] @ tau_t + tau_t @ p[b, t]
            u[b, t] = ut
            xt = A[b, t] @ xt + B[b, t] @ ut + c1[b, t]
            x[b, t + 1] = xt
        cost[b] = c
    return x, u, cost, xtr, st


def lqr_bwd(Q, p, A, B, c1, x_init, x, u, gx, gu, gc):
    """Adjoint of `lqr` at its solution (x, u): gradients of <gx, x> + <gu, u> + <gc, cost> with respect to the
    full-size Q, p, A, B, c1 and x_init.  The gradient with respect to u_traj is 0 (the minimiser does not depend on it).

    One more LQR solve with the same Q_t, F_t, the linear term -g_tau and the terminal term -gx_T from a zero initial
    state gives d_tau; the duals of the solution (lam) and of the adjoint (dlam) follow backwards, and
      dQ_t = -sym(d_tau tau^T) + gc tau tau^T / 2,  dp_t = -d_tau + gc tau,
      dF_t = -(lam_{t+1} d_tau^T + dlam_{t+1} tau^T),  dc1_t = -dlam_{t+1},  dx_init = -dlam_0.
    dQ_t is the symmetric gradient: the problem depends on Q only through its symmetric part, and the antisymmetric part
    of autograd through the reference's recursion depends on u_traj."""
    nb, T, n = p.shape
    ns = x_init.shape[-1]
    out = [np.zeros(Q.shape), np.zeros(p.shape), np.zeros(A.shape), np.zeros(B.shape), np.zeros(c1.shape),
           np.zeros(x_init.shape)]
    gQ, gp, gA, gB, gc1, gx0 = out
    for b in range(nb):
        tau = np.concatenate([x[b, :T], u[b]], -1)
        g = np.concatenate([gx[b, :T], gu[b]], -1) + gc[b] * (np.einsum('tij,tj->ti', Q[b], tau) + p[b])
        Qts, _, _ = _riccati(Q[b], A[b], B[b], ns)
        ks = _gains(Qts, lambda t: -g[t], A[b], B[b], ns, vT=-gx[b, T])
        dtau = np.zeros((T, n))
        dx = np.zeros(ns)
        for t in range(T):
            du = Qts[t][1] @ dx + ks[t]
            dtau[t] = np.concatenate([dx, du])
            dx = np.concatenate([A[b, t], B[b, t]], -1) @ dtau[t]
        lam, dlam = np.zeros(ns), -gx[b, T]
        for t in range(T - 1, -1, -1):
            dF = -(np.outer(lam, dtau[t]) + np.outer(dlam, tau[t]))
            gA[b, t], gB[b, t] = dF[:, :ns], dF[:, ns:]
            gc1[b, t] = -dlam
            gQ[b, t] = -0.5 * (np.outer(dtau[t], tau[t]) + np.outer(tau[t], dtau[t])) + 0.5 * gc[b] * np.outer(tau[t], tau[t])
            gp[b, t] = -dtau[t] + gc[b] * tau[t]
            F = np.concatenate([A[b, t], B[b, t]], -1)
            lam_n = (Q[b, t] @ tau[t] + p[b, t] + F.T @ lam)[:ns]
            dlam = (Q[b, t] @ dtau[t] + F.T @ dlam - g[t])[:ns]
            lam = lam_n
        gx0[b] = -dlam
    return out
