"""Trajectories of the REFERENCE's dense LM (pypose v0.9.5, fp64, CPU) on its examples/module/pgo `PoseGraph` with SO3
nodes, r_e = Log(Z_e^-1 A^-1 B), on synthetic rotation-averaging view graphs (oracle/so3pgo_oracle.py problem: random
absolute rotations, about 6 relative rotations per camera, a start perturbed from the truth):

    constant     Constant(damping=1e-6)
    trustregion  TrustRegion()
    far          TrustRegion() from a far start (errors up to 2.5 rad)
    huber        TrustRegion() with a Huber kernel (delta 0.05)
    cauchy       TrustRegion() with a Cauchy kernel (delta 0.1)
    module       TrustRegion() on a second, denser graph (the user-module form of the tests)

and the reference's autograd Jacobians d r / d B of single edges, with residual angles from 0 to pi - 1e-3 (`jac/*`;
`jac/J4` is the reference's full 4-column Jacobian, whose 4th column is zero).
    PYPOSE_REFERENCE=<reference checkout> python oracle/make_golden_so3pgo.py     # writes tests/golden/so3pgo.npz
Test infrastructure only.
"""
import os
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "so3pgo.npz")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import lie_oracle as L  # noqa: E402
from oracle.so3pgo_oracle import problem  # noqa: E402


class PoseGraph(nn.Module):
    def __init__(self, nodes):
        super().__init__()
        self.nodes = ref.Parameter(nodes)

    def forward(self, edges, poses):
        node1 = self.nodes[edges[..., 0]]
        node2 = self.nodes[edges[..., 1]]
        error = poses.Inv() @ node1.Inv() @ node2
        return error.Log().tensor()


CASES = {
    # name: (problem kwargs, strategy, steps, kernel)
    "constant": (dict(seed=0), "constant", 5, None),
    "trustregion": (dict(seed=1, far=0.3), "trustregion", 5, None),
    "far": (dict(seed=2, far=1.5), "trustregion", 8, None),
    "huber": (dict(seed=3, far=0.3), "trustregion", 5, ("huber", 0.05)),
    "cauchy": (dict(seed=4, far=0.3), "trustregion", 5, ("cauchy", 0.1)),
    "module": (dict(seed=5, N=120, deg=10, far=0.3), "trustregion", 5, None),
}


def run(kw, kind, steps, kernel):
    d = problem(**kw)
    edges, Z = torch.from_numpy(d["edges"]), ref.SO3(torch.from_numpy(d["Z"]))
    model = PoseGraph(ref.SO3(torch.from_numpy(d["nodes0"]).clone()))
    strategy = ref.optim.strategy.Constant(damping=1e-6) if kind == "constant" else ref.optim.strategy.TrustRegion()
    if kernel is None:
        k = None
    elif kernel[0] == "huber":
        k = ref.optim.kernel.Huber(delta=kernel[1])
    else:
        k = ref.optim.kernel.Cauchy(delta=kernel[1])
    opt = ref.optim.LM(model, strategy=strategy, kernel=k, reject=16)
    loss, nodes, rej = [], [], []
    for _ in range(steps):
        loss.append(float(opt.step(input=(edges, Z))))
        nodes.append(model.nodes.detach().tensor().numpy().copy())
        rej.append(opt.reject_count)
    out = dict(d)
    out.update(loss=np.array(loss), nodes=np.stack(nodes), reject=np.array(rej))
    return out


def jacobians(seed=7):
    """Single edges (A, B, Z) with |r| from 0 to pi - 1e-3 and the reference's d r / d B (4 columns; J = the first 3)."""
    rng = np.random.default_rng(seed)
    angles = np.concatenate([[0.0, 1e-12, 1e-8, 1e-5, 1e-3], np.geomspace(1e-2, 3.0, 18), [np.pi - 1e-3]])
    n = len(angles)
    A = ref.randn_SO3(n, sigma=1.0)
    B = ref.randn_SO3(n, sigma=1.0)
    axis = rng.normal(0, 1, (n, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    noise = ref.so3(torch.from_numpy(axis * angles[:, None]))
    Z = (A.Inv() @ B) @ noise.Exp().Inv()                      # r = Log(Z^-1 A^-1 B) = noise
    Js = []
    for e in range(n):
        def f(b):
            return (Z[e].Inv() @ A[e].Inv() @ ref.SO3(b)).Log().tensor()
        Bp = ref.Parameter(B[e].clone())
        Js.append(torch.autograd.functional.jacobian(lambda t: f(t), Bp.tensor()).numpy())
    J4 = np.stack(Js)
    r = (Z.Inv() @ A.Inv() @ B).Log().tensor().numpy()
    return dict(A=A.tensor().numpy(), B=B.tensor().numpy(), Z=Z.tensor().numpy(), r=r, J=J4[..., :3], J4=J4)


def main():
    torch.set_default_dtype(torch.float64)
    torch.manual_seed(0)
    arrays = {}
    for name, (kw, kind, steps, kernel) in CASES.items():
        r = run(kw, kind, steps, kernel)
        print(name, "N", len(r["nodes0"]), "E", len(r["edges"]), "loss", r["loss"], "reject", r["reject"])
        for k, v in r.items():
            arrays[f"{name}/{k}"] = v
    for k, v in jacobians().items():
        arrays[f"jac/{k}"] = v
    print("jac |r|", np.linalg.norm(arrays["jac/r"], axis=1)[[0, -1]])
    err0 = L.log("SO3", L.mul("SO3", arrays["far/nodes0"], L.inv("SO3", arrays["far/gt"])))
    assert np.linalg.norm(err0, axis=1).max() > 2.0, "the far start must be far"
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
