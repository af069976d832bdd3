"""fp64 numpy restatement of the Sim3 pose-graph route (csrc/sim3pgo_math.cuh, csrc/sim3pgo.cu, the width-7 kernels of
csrc/pcg2.cu, optim/structured.py Sim3PGOProblem) and of the reference's dense LM on the same model
(pypose/optim/optimizer.py:645-680, 8 dense columns per Sim3 node).

    r_e = Log(Z_e^-1 A^-1 B),   A = nodes[i], B = nodes[j],   r = [tau(3) phi(3) sigma]
    J_B = sim3_Jl_inv(r) Sim3_Adj(Z^-1 A^-1)   (the reference's truncated series, operation.py:167-172),   J_A = -J_B

Test infrastructure only.
"""
import numpy as np

from oracle import lie_oracle as L
from oracle.lm_oracle import node_layout, robust


def problem(seed, N=12, loops=3, drift=0.03, noise=0.01, far=1.0):
    """A synthetic monocular-drift graph: a ground-truth trajectory (unit scale), an odometry chain whose relative scale
    drifts slowly (e^(drift k) at step k) with noise, `loops` loop closures measured at unit scale, and a start built by
    chaining the drifted odometry (`far` scales the odometry noise of the start).  Returns nodes0 (N,8), edges (E,2),
    Z (E,8) and the ground truth."""
    rng = np.random.default_rng(seed)
    steps = np.concatenate([rng.normal([1.0, 0.0, 0.0], 0.1, (N - 1, 3)), rng.normal(0, 0.15, (N - 1, 3)),
                            np.zeros((N - 1, 1))], 1)
    gt = [L.exp("Sim3", np.zeros(7))]
    for k in range(N - 1):
        gt.append(L.mul("Sim3", gt[-1], L.exp("Sim3", steps[k])))
    gt = np.stack(gt)
    ij = [(k, k + 1) for k in range(N - 1)]
    while len(ij) < N - 1 + loops:
        a, b = sorted(rng.choice(N, 2, replace=False))
        if b - a > 2 and (a, b) not in ij:
            ij.append((a, b))
    edges = np.array(ij, np.int64)
    rel = L.mul("Sim3", L.inv("Sim3", gt[edges[:, 0]]), gt[edges[:, 1]])
    n = rng.normal(0, noise, (len(edges), 7))
    n[: N - 1, 6] += drift * np.arange(1, N)                   # odometry: slowly drifting relative scale
    Z = L.mul("Sim3", rel, L.exp("Sim3", n))
    # start: the drifted odometry chained from node 0, plus extra noise
    g = np.random.default_rng(100 + seed)
    nodes0 = [gt[0]]
    for k in range(N - 1):
        nodes0.append(L.mul("Sim3", nodes0[-1], L.mul("Sim3", Z[k], L.exp("Sim3", g.normal(0, 0.02 * far, 7)))))
    return dict(nodes0=np.stack(nodes0), edges=edges, Z=Z, gt=gt)


def residual(nodes, Z, edges):
    """r (E,7) and S = Z^-1 A^-1 (E,8)."""
    S = L.mul("Sim3", L.inv("Sim3", Z), L.inv("Sim3", nodes[edges[:, 0]]))
    return L.log("Sim3", L.mul("Sim3", S, nodes[edges[:, 1]])), S


def jacobian(nodes, Z, edges):
    """J_B (E,7,7) = sim3_Jl_inv(r) Sim3_Adj(S) and r (E,7)."""
    r, S = residual(nodes, Z, edges)
    return L.sim3_Jl_inv(r) @ L.Sim3_Adj(S), r


def blocks(nodes, Z, edges, kind=0, delta=1.0):
    """Per-edge M (E,7,7) = w J^T J, u (E,7) = w J^T r (FastTriggs weight w = rho'), the loss and J, r."""
    J, r = jacobian(nodes, Z, edges)
    rho, w = robust(kind, delta, (r * r).sum(-1))
    M = w[:, None, None] * np.swapaxes(J, 1, 2) @ J
    u = w[:, None] * np.einsum("eka,ek->ea", J, r)
    return dict(M=M, u=u, loss=rho.sum(), J=J, r=r, w=w)


def pack(M):
    """Row-major upper triangle of (..., 7, 7) -> (..., 28)."""
    iu = np.triu_indices(7)
    return M[..., iu[0], iu[1]]


def node_blocks(b, edges, N):
    """Node-ordered slots: Mn (2E,28) with the edge's block at both endpoints' slots, un (2E,7) = -u / +u, and the layout
    (epos_i, epos_j, nptr, nother)."""
    ei, ej = edges[:, 0], edges[:, 1]
    epos_i, epos_j, nptr, nother = node_layout(ei, ej, N)
    Mn, un = np.zeros((2 * len(ei), 28)), np.zeros((2 * len(ei), 7))
    Mn[epos_i] = Mn[epos_j] = pack(b["M"])
    un[epos_i], un[epos_j] = -b["u"], b["u"]
    return Mn, un, (epos_i, epos_j, nptr, nother)


def node_sums(b, edges, N):
    """Hd (N,7,7) = sum of the node's blocks, g (N,7) = sum of its signed u."""
    Hd, g = np.zeros((N, 7, 7)), np.zeros((N, 7))
    for s, k in ((-1.0, 0), (1.0, 1)):
        np.add.at(Hd, edges[:, k], b["M"])
        np.add.at(g, edges[:, k], s * b["u"])
    return Hd, g


def dense_H(b, edges, N):
    """The (7N,7N) J^T J of the graph: M_e on (i,i), (j,j), -M_e on (i,j), (j,i)."""
    H = np.zeros((7 * N, 7 * N))
    for e, (i, j) in enumerate(edges):
        for a, c, s in ((i, i, 1), (j, j, 1), (i, j, -1), (j, i, -1)):
            H[7 * a:7 * a + 7, 7 * c:7 * c + 7] += s * b["M"][e]
    return H


def damp(Hd, scale, dmin=1e-6, dmax=1e32):
    """(damped blocks, extra (N,7) added to the diagonal)."""
    d = np.diagonal(Hd, axis1=1, axis2=2)
    c = np.clip(d, dmin, dmax) * scale
    H = Hd.copy()
    i = np.arange(7)
    H[:, i, i] = c
    return H, c - d


def loss(nodes, Z, edges, kind=0, delta=1.0):
    r, _ = residual(nodes, Z, edges)
    return robust(kind, delta, (r * r).sum(-1))[0].sum()


def retract(nodes, D):
    """Exp(D) nodes for D (N,7): Sim3Type.add_ of the reference (the 8th step component is dropped)."""
    return L.mul("Sim3", L.exp("Sim3", D), nodes)


def dense_step(nodes, Z, edges, scale, kind=0, delta=1.0, dmin=1e-6, dmax=1e32):
    """The reference's dense damped step with 8 columns per node (the 8th identically zero): A = J^T J with the diagonal
    clamped and scaled, D = A^-1 (-J^T R).  Returns D (N,8), the predicted reduction and the current loss."""
    N, E = len(nodes), len(edges)
    b = blocks(nodes, Z, edges, kind, delta)
    sw = np.sqrt(b["w"])
    J = np.zeros((7 * E, 8 * N))
    for e, (i, j) in enumerate(edges):
        J[7 * e:7 * e + 7, 8 * i:8 * i + 7] -= sw[e] * b["J"][e]
        J[7 * e:7 * e + 7, 8 * j:8 * j + 7] += sw[e] * b["J"][e]
    R = (sw[:, None] * b["r"]).reshape(-1)
    A = J.T @ J
    k = np.arange(8 * N)
    A[k, k] = np.clip(A[k, k], dmin, dmax) * scale
    D = np.linalg.solve(A, -J.T @ R)
    Jd = J @ D
    return D.reshape(N, 8), float(Jd @ (2 * R + Jd)), b["loss"]


def lm(nodes, Z, edges, steps, strategy="constant", damping=1e-6, reject=16, kind=0, delta=1.0):
    """The reference's dense LM (optimizer.py:659-680) with Constant(damping) or TrustRegion() (strategy.py) in fp64."""
    tr = dict(down=0.5)
    dmp = 1e-6 if strategy == "trustregion" else damping
    hist, Ns, rej = [], [], []
    last = None
    for _ in range(steps):
        cur = None
        scale, nrej = 1.0, 0
        while True:
            scale *= 1 + dmp
            D, pred, l0 = dense_step(nodes, Z, edges, scale, kind, delta)
            cur = l0 if last is None else last
            trial = retract(nodes, D[:, :7])
            lt = loss(trial, Z, edges, kind, delta)
            if strategy == "trustregion":                       # strategy.py TrustRegion.update
                quality = (cur - lt) / -pred
                radius = 1.0 / dmp
                if quality > 0.5:
                    radius, tr["down"] = 2.0 * radius, 0.5
                elif quality > 1e-3:
                    tr["down"] = 0.5
                else:
                    radius, tr["down"] = radius * tr["down"], tr["down"] * 0.5
                tr["down"] = max(1e-6, min(tr["down"], 1e16))
                dmp = 1.0 / max(1e-6, min(radius, 1e16))
            if cur < lt and nrej < reject:
                nrej += 1
                continue
            nodes, last = trial, lt
            break
        hist.append(last); Ns.append(nodes); rej.append(nrej)
    return dict(loss=np.array(hist), nodes=np.stack(Ns), reject=np.array(rej))
