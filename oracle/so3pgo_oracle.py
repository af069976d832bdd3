"""fp64 numpy restatement of the SO3 pose-graph route (rotation averaging: csrc/so3pgo_math.cuh, csrc/so3pgo.cu, the
width-3 kernels of csrc/pcg2.cu, optim/structured.py SO3PGOProblem) and of the reference's dense LM on the same model
(pypose/optim/optimizer.py:645-680, 4 dense columns per SO3 node).

    r_e = Log(Z_e^-1 A^-1 B),   A = nodes[i], B = nodes[j],   r in R^3
    J_B = so3_Jl_inv(r) SO3_Adj(Z^-1 A^-1)   (operation.py:23-32; SO3_Adj is the rotation matrix),   J_A = -J_B

Test infrastructure only.
"""
import numpy as np

from oracle import lie_oracle as L
from oracle.lm_oracle import node_layout, robust


def problem(seed, N=60, deg=6, noise=0.02, far=0.1, max_start=2.5):
    """A synthetic rotation-averaging view graph: N random absolute rotations, a chain (k, k+1) for connectivity plus
    random pairs up to about `deg` edges per node, relative rotations Z_ij = R_i^-1 R_j Exp(n) with noise `noise`, and a
    start Exp(d) R_i with |d| ~ `far` (clipped to `max_start` rad).  Returns nodes0 (N,4), edges (E,2), Z (E,4), gt."""
    rng = np.random.default_rng(seed)
    gt = L.exp("SO3", rng.normal(0, 1.0, (N, 3)))
    ij = {(k, k + 1) for k in range(N - 1)}
    E = max(N - 1, N * deg // 2)
    while len(ij) < E:
        a, b = sorted(rng.choice(N, 2, replace=False))
        ij.add((int(a), int(b)))
    edges = np.array(sorted(ij), np.int64)
    edges = edges[rng.permutation(len(edges))]
    rel = L.mul("SO3", L.inv("SO3", gt[edges[:, 0]]), gt[edges[:, 1]])
    Z = L.mul("SO3", rel, L.exp("SO3", rng.normal(0, noise, (len(edges), 3))))
    d = rng.normal(0, far, (N, 3))
    n = np.linalg.norm(d, axis=1, keepdims=True)
    d = np.where(n > max_start, d * max_start / np.maximum(n, 1e-300), d)
    nodes0 = L.mul("SO3", L.exp("SO3", d), gt)
    return dict(nodes0=nodes0, edges=edges, Z=Z, gt=gt)


def residual(nodes, Z, edges):
    """r (E,3) and S = Z^-1 A^-1 (E,4)."""
    S = L.mul("SO3", L.inv("SO3", Z), L.inv("SO3", nodes[edges[:, 0]]))
    return L.log("SO3", L.mul("SO3", S, nodes[edges[:, 1]])), S


def jacobian(nodes, Z, edges):
    """J_B (E,3,3) = so3_Jl_inv(r) SO3_Adj(S) and r (E,3)."""
    r, S = residual(nodes, Z, edges)
    return L.so3_Jl_inv(r) @ L.SO3_Adj(S), r


def blocks(nodes, Z, edges, kind=0, delta=1.0):
    """Per-edge M (E,3,3) = w J^T J, u (E,3) = w J^T r (FastTriggs weight w = rho'), the loss and J, r."""
    J, r = jacobian(nodes, Z, edges)
    rho, w = robust(kind, delta, (r * r).sum(-1))
    M = w[:, None, None] * np.swapaxes(J, 1, 2) @ J
    u = w[:, None] * np.einsum("eka,ek->ea", J, r)
    return dict(M=M, u=u, loss=rho.sum(), J=J, r=r, w=w)


def pack(M):
    """Row-major upper triangle of (..., 3, 3) -> (..., 6)."""
    iu = np.triu_indices(3)
    return M[..., iu[0], iu[1]]


def node_blocks(b, edges, N):
    """Node-ordered slots: Mn (2E,8) with the edge's packed block (6 words, then 2 zero words) at both endpoints' slots,
    un (2E,3) = -u / +u, and the layout (epos_i, epos_j, nptr, nother)."""
    ei, ej = edges[:, 0], edges[:, 1]
    epos_i, epos_j, nptr, nother = node_layout(ei, ej, N)
    Mn, un = np.zeros((2 * len(ei), 8)), np.zeros((2 * len(ei), 3))
    Mn[epos_i, :6] = Mn[epos_j, :6] = pack(b["M"])
    un[epos_i], un[epos_j] = -b["u"], b["u"]
    return Mn, un, (epos_i, epos_j, nptr, nother)


def node_sums(b, edges, N):
    """Hd (N,3,3) = sum of the node's blocks, g (N,3) = sum of its signed u."""
    Hd, g = np.zeros((N, 3, 3)), np.zeros((N, 3))
    for s, k in ((-1.0, 0), (1.0, 1)):
        np.add.at(Hd, edges[:, k], b["M"])
        np.add.at(g, edges[:, k], s * b["u"])
    return Hd, g


def dense_H(b, edges, N):
    """The (3N,3N) J^T J of the graph: M_e on (i,i), (j,j), -M_e on (i,j), (j,i)."""
    H = np.zeros((3 * N, 3 * N))
    for e, (i, j) in enumerate(edges):
        for a, c, s in ((i, i, 1), (j, j, 1), (i, j, -1), (j, i, -1)):
            H[3 * a:3 * a + 3, 3 * c:3 * c + 3] += s * b["M"][e]
    return H


def damp(Hd, scale, dmin=1e-6, dmax=1e32):
    """(damped blocks, extra (N,3) added to the diagonal)."""
    d = np.diagonal(Hd, axis1=1, axis2=2)
    c = np.clip(d, dmin, dmax) * scale
    H = Hd.copy()
    i = np.arange(3)
    H[:, i, i] = c
    return H, c - d


def loss(nodes, Z, edges, kind=0, delta=1.0):
    r, _ = residual(nodes, Z, edges)
    return robust(kind, delta, (r * r).sum(-1))[0].sum()


def retract(nodes, D):
    """Exp(D) nodes for D (N,3): SO3Type.add_ of the reference (the 4th step component is dropped)."""
    return L.mul("SO3", L.exp("SO3", D), nodes)


def dense_step(nodes, Z, edges, scale, kind=0, delta=1.0, dmin=1e-6, dmax=1e32):
    """The reference's dense damped step with 4 columns per node (the 4th identically zero): A = J^T J with the diagonal
    clamped and scaled, D = A^-1 (-J^T R).  Returns D (N,4), the predicted reduction and the current loss."""
    N, E = len(nodes), len(edges)
    b = blocks(nodes, Z, edges, kind, delta)
    sw = np.sqrt(b["w"])
    J = np.zeros((3 * E, 4 * N))
    for e, (i, j) in enumerate(edges):
        J[3 * e:3 * e + 3, 4 * i:4 * i + 3] -= sw[e] * b["J"][e]
        J[3 * e:3 * e + 3, 4 * j:4 * j + 3] += sw[e] * b["J"][e]
    R = (sw[:, None] * b["r"]).reshape(-1)
    A = J.T @ J
    k = np.arange(4 * N)
    A[k, k] = np.clip(A[k, k], dmin, dmax) * scale
    D = np.linalg.solve(A, -J.T @ R)
    Jd = J @ D
    return D.reshape(N, 4), float(Jd @ (2 * R + Jd)), b["loss"]


def lm(nodes, Z, edges, steps, strategy="constant", damping=1e-6, reject=16, kind=0, delta=1.0):
    """The reference's dense LM (optimizer.py:659-680) with Constant(damping) or TrustRegion() (strategy.py) in fp64."""
    tr = dict(down=0.5)
    dmp = 1e-6 if strategy == "trustregion" else damping
    hist, Ns, rej = [], [], []
    last = None
    for _ in range(steps):
        scale, nrej = 1.0, 0
        while True:
            scale *= 1 + dmp
            D, pred, l0 = dense_step(nodes, Z, edges, scale, kind, delta)
            cur = l0 if last is None else last
            trial = retract(nodes, D[:, :3])
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
