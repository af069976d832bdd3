"""Trajectories of the REFERENCE's dense LM (pypose v0.9.5, fp64, CPU) on its examples/module/pgo `PoseGraph` with Sim3
nodes, r_e = Log(Z_e^-1 A^-1 B), on synthetic monocular-drift graphs (oracle/sim3pgo_oracle.py problem: an odometry chain
whose relative scale drifts slowly, loop closures at unit scale, a start chained from the drifted odometry):

    constant     Constant(damping=1e-6)
    trustregion  TrustRegion()
    reject       TrustRegion() from a far start, with rejected trials
    huber        TrustRegion() with a Huber kernel (delta 0.05)
    module       TrustRegion() on a second graph (the user-module form of the tests)

and the reference's autograd Jacobians d r / d B of single edges, with residual norms from 1e-3 to about 5 (`jac/*`).
    PYPOSE_REFERENCE=<reference checkout> python oracle/make_golden_sim3pgo.py     # writes tests/golden/sim3pgo.npz
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

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "sim3pgo.npz")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.sim3pgo_oracle import problem  # noqa: E402


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
    # name: (seed, strategy, steps, far, kernel)
    "constant": (0, "constant", 5, 1.0, None),
    "trustregion": (1, "trustregion", 5, 1.0, None),
    "reject": (2, "trustregion", 8, 80.0, None),
    "huber": (3, "trustregion", 5, 3.0, 0.05),
    "module": (4, "trustregion", 5, 1.0, None),
}


def run(seed, kind, steps, far, huber):
    d = problem(seed, far=far)
    edges, Z = torch.from_numpy(d["edges"]), ref.Sim3(torch.from_numpy(d["Z"]))
    model = PoseGraph(ref.Sim3(torch.from_numpy(d["nodes0"]).clone()))
    strategy = ref.optim.strategy.Constant(damping=1e-6) if kind == "constant" else ref.optim.strategy.TrustRegion()
    kernel = ref.optim.kernel.Huber(delta=huber) if huber else None
    opt = ref.optim.LM(model, strategy=strategy, kernel=kernel, reject=16)
    loss, nodes, rej = [], [], []
    for _ in range(steps):
        loss.append(float(opt.step(input=(edges, Z))))
        nodes.append(model.nodes.detach().tensor().numpy().copy())
        rej.append(opt.reject_count)
    out = dict(d)
    out.update(loss=np.array(loss), nodes=np.stack(nodes), reject=np.array(rej))
    return out


def jacobians(seed=7, n=24):
    """Single edges (A, B, Z) with |r| spread over 1e-3 .. ~5 and the reference's d r / d B (7 tangent columns)."""
    rng = np.random.default_rng(seed)
    A = ref.randn_Sim3(n, sigma=1.0)
    B = ref.randn_Sim3(n, sigma=1.0)
    size = torch.from_numpy(np.geomspace(1e-3, 1.6, n))[:, None]
    noise = ref.sim3(torch.from_numpy(rng.normal(0, 1, (n, 7))) * size)
    Z = (A.Inv() @ B) @ noise.Exp().Inv()                      # r = Log(Z^-1 A^-1 B) = noise
    Js = []
    for e in range(n):
        def f(b):
            return (Z[e].Inv() @ A[e].Inv() @ ref.Sim3(b)).Log().tensor()
        Bp = ref.Parameter(B[e].clone())
        J = torch.autograd.functional.jacobian(lambda t: f(t), Bp.tensor())
        Js.append(J[:, :7].numpy())
    r = (Z.Inv() @ A.Inv() @ B).Log().tensor().numpy()
    return dict(A=A.tensor().numpy(), B=B.tensor().numpy(), Z=Z.tensor().numpy(), r=r, J=np.stack(Js))


def main():
    torch.set_default_dtype(torch.float64)
    torch.manual_seed(0)
    arrays = {}
    for name, (seed, kind, steps, far, huber) in CASES.items():
        r = run(seed, kind, steps, far, huber)
        print(name, "loss", r["loss"], "reject", r["reject"])
        for k, v in r.items():
            arrays[f"{name}/{k}"] = v
    for k, v in jacobians().items():
        arrays[f"jac/{k}"] = v
    print("jac |r|", np.linalg.norm(arrays["jac/r"], axis=1)[[0, -1]])
    assert arrays["reject/reject"].sum() > 0, "the far start must reject at least one trial"
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
