"""Generate golden vectors by running the REFERENCE itself (pypose v0.9.5 imported from
the checkout named by PYPOSE_REFERENCE) in fp64 on CPU:

    python oracle/make_golden.py            # writes tests/golden/lie_ops.npz

The tests read only the committed .npz, never the reference.  Inputs are seeded; every
(group, op) gets N_RANDOM random rows plus hand-placed edge rows (identity, tiny / near-pi angles,
negative-w quaternions).  Backward goldens come from the reference's own autograd.
"""
import os
import sys

import numpy as np
import torch

REF = os.environ["PYPOSE_REFERENCE"]
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402
from pypose.lietensor import operation as rop  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
N_RANDOM = 48
DT = torch.float64

GROUPS = {"SO3": ("so3", 4, 3), "SE3": ("se3", 7, 6), "RxSO3": ("rxso3", 5, 4), "Sim3": ("sim3", 8, 7)}
RANDN_ALG = {"SO3": ref.randn_so3, "SE3": ref.randn_se3, "RxSO3": ref.randn_rxso3, "Sim3": ref.randn_sim3}
EXP = {"SO3": rop.so3_Exp, "SE3": rop.se3_Exp, "RxSO3": rop.rxso3_Exp, "Sim3": rop.sim3_Exp}
LOG = {"SO3": rop.SO3_Log, "SE3": rop.SE3_Log, "RxSO3": rop.RxSO3_Log, "Sim3": rop.Sim3_Log}
INV = {"SO3": rop.SO3_Inv, "SE3": rop.SE3_Inv, "RxSO3": rop.RxSO3_Inv, "Sim3": rop.Sim3_Inv}
MUL = {"SO3": rop.SO3_Mul, "SE3": rop.SE3_Mul, "RxSO3": rop.RxSO3_Mul, "Sim3": rop.Sim3_Mul}
ACT = {"SO3": rop.SO3_Act, "SE3": rop.SE3_Act, "RxSO3": rop.RxSO3_Act, "Sim3": rop.Sim3_Act}
ACT4 = {"SO3": rop.SO3_Act4, "SE3": rop.SE3_Act4, "RxSO3": rop.RxSO3_Act4, "Sim3": rop.Sim3_Act4}
ADJ = {"SO3": rop.SO3_AdjXa, "SE3": rop.SE3_AdjXa, "RxSO3": rop.RxSO3_AdjXa, "Sim3": rop.Sim3_AdjXa}
ADJT = {"SO3": rop.SO3_AdjTXa, "SE3": rop.SE3_AdjTXa, "RxSO3": rop.RxSO3_AdjTXa, "Sim3": rop.Sim3_AdjTXa}
LTYPE = {"SO3": ref.SO3_type, "SE3": ref.SE3_type, "RxSO3": ref.RxSO3_type, "Sim3": ref.Sim3_type}


def rot_part(grp):
    return {"SO3": slice(0, 3), "SE3": slice(3, 6), "RxSO3": slice(0, 3), "Sim3": slice(3, 6)}[grp]


def algebra_inputs(grp, gen):
    """random algebra rows (angle spread over (0, pi)) + edge rows."""
    K = GROUPS[grp][2]
    x = RANDN_ALG[grp](N_RANDOM, dtype=DT).tensor()
    # re-scale rotation angles to U(0, pi - 1e-3) so Exp/Log round trips are well defined
    r = rot_part(grp)
    phi = x[:, r]
    ang = torch.rand(N_RANDOM, 1, dtype=DT) * (np.pi - 1e-3)
    x[:, r] = phi / phi.norm(dim=-1, keepdim=True) * ang
    edges = []
    axis = torch.tensor([0.6, -0.48, 0.64], dtype=DT)
    for a in (0.0, 1e-12, 1e-8, 1e-4, 1e-2, 0.3, 1.5, np.pi - 1e-6, np.pi - 1e-3):
        e = torch.randn(K, dtype=DT) * 0.7
        e[r] = axis * a
        edges.append(e)
    z = torch.zeros(K, dtype=DT)
    edges.append(z)
    if grp in ("RxSO3", "Sim3"):           # zero scale-log with non-trivial rotation
        e = torch.randn(K, dtype=DT) * 0.7
        e[-1] = 0.0
        edges.append(e)
    return torch.cat([x, torch.stack(edges)], 0)


def group_inputs(grp):
    x = algebra_inputs(grp, None)
    X = EXP[grp].apply(x)
    # flip the quaternion sign of some rows (w < 0 is legal and not canonicalised by Log)
    q = {"SO3": slice(0, 4), "SE3": slice(3, 7), "RxSO3": slice(0, 4), "Sim3": slice(3, 7)}[grp]
    X = X.clone()
    X[::5, q] = -X[::5, q]
    return X


def main():
    torch.manual_seed(20260922)
    os.makedirs(OUT, exist_ok=True)
    gold = {}

    def put(key, ins, outs):
        for i, t in enumerate(ins):
            gold[f"{key}/in{i}"] = t.detach().numpy().copy()
        for i, t in enumerate(outs):
            gold[f"{key}/out{i}"] = t.detach().numpy().copy()

    for grp, (alg, D, K) in GROUPS.items():
        # Exp fwd/bwd
        x = algebra_inputs(grp, None).requires_grad_(True)
        X = EXP[grp].apply(x)
        gX = torch.randn_like(X)
        (gx,) = torch.autograd.grad(X, x, gX)
        put(f"{alg}_exp_fwd", [x], [X])
        put(f"{alg}_exp_bwd", [x, gX], [gx])
        # Log fwd/bwd
        Xg = group_inputs(grp).requires_grad_(True)
        xo = LOG[grp].apply(Xg)
        g = torch.randn_like(xo)
        (gXg,) = torch.autograd.grad(xo, Xg, g)
        put(f"{grp}_log_fwd", [Xg], [xo])
        put(f"{grp}_log_bwd", [xo, g], [gXg])
        # Inv
        Xg = group_inputs(grp).requires_grad_(True)
        Y = INV[grp].apply(Xg)
        gY = torch.randn_like(Y)
        (gXg,) = torch.autograd.grad(Y, Xg, gY)
        put(f"{grp}_inv_fwd", [Xg], [Y])
        put(f"{grp}_inv_bwd", [Y, gY], [gXg])
        # Mul
        A = group_inputs(grp).requires_grad_(True)
        B = group_inputs(grp)[torch.randperm(A.shape[0])].requires_grad_(True)
        Z = MUL[grp].apply(A, B)
        gZ = torch.randn_like(Z)
        gA, gB = torch.autograd.grad(Z, (A, B), gZ)
        put(f"{grp}_mul_fwd", [A, B], [Z])
        put(f"{grp}_mul_bwd", [A, gZ], [gA, gB])
        # Act / Act4
        for name, FN, w in (("act", ACT, 3), ("act4", ACT4, 4)):
            A = group_inputs(grp).requires_grad_(True)
            p = torch.randn(A.shape[0], w, dtype=DT, requires_grad=True)
            o = FN[grp].apply(A, p)
            g = torch.randn_like(o)
            gA, gp = torch.autograd.grad(o, (A, p), g)
            put(f"{grp}_{name}_fwd", [A, p], [o])
            put(f"{grp}_{name}_bwd", [A, o, g], [gA, gp])
        # Adj
        A = group_inputs(grp).requires_grad_(True)
        a = torch.randn(A.shape[0], K, dtype=DT, requires_grad=True)
        o = ADJ[grp].apply(A, a)
        g = torch.randn_like(o)
        gA, ga = torch.autograd.grad(o, (A, a), g)
        put(f"{grp}_adj_fwd", [A, a], [o])
        put(f"{grp}_adj_bwd", [A, o, g], [gA, ga])
        # AdjT
        A = group_inputs(grp).requires_grad_(True)
        a = torch.randn(A.shape[0], K, dtype=DT, requires_grad=True)
        o = ADJT[grp].apply(A, a)
        g = torch.randn_like(o)
        gA, ga = torch.autograd.grad(o, (A, a), g)
        put(f"{grp}_adjt_fwd", [A, a], [o])
        put(f"{grp}_adjt_bwd", [A, a, g], [gA, ga])
        # Jinvp (through the LieTensor API, as the reference has no Function for it) + its autograd
        A = group_inputs(grp).requires_grad_(True)
        p = torch.randn(A.shape[0], K, dtype=DT, requires_grad=True)
        o = ref.LieTensor(A, ltype=LTYPE[grp]).Jinvp(p).tensor()
        g = torch.randn_like(o)
        gA, gp = torch.autograd.grad(o, (A, p), g)
        put(f"{grp}_jinvp_fwd", [A, p], [o])
        put(f"{grp}_jinvp_grad", [A, p, g], [gA, gp])

    # so3 Jr
    x = algebra_inputs("SO3", None)
    J = ref.so3(x).Jr()
    put("so3_jr", [x], [J.reshape(-1, 9)])

    path = os.path.join(OUT, "lie_ops.npz")
    np.savez_compressed(path, **gold)
    print("wrote", path, len(gold), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
