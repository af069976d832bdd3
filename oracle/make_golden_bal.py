"""Trajectories of the REFERENCE's dense LM (pypose v0.9.5, fp64, CPU) on the BAL model of its
examples/module/ba/bundle_adjustment.py (`Reproj(K, C, P)`, without `@psjac`, which needs the `bae` package):

    y = T_c p_j,   n = -y[:2] / y[2],   r = f (1 + k1 |n|^2 + k2 |n|^4) n - z

8 cameras, 60 points, 400 observations, f ~ 500, |k1| <= 0.1, |k2| <= 0.01, points 3-8 units in front of the cameras
(BAL convention: the camera looks down -z).  Constant and TrustRegion strategies from a perturbed start, and one
TrustRegion run from a far start with rejected trials.
    PYPOSE_REFERENCE=<reference checkout> python oracle/make_golden_bal.py      # writes tests/golden/bal.npz
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

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "bal.npz")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.bal_oracle import problem  # noqa: E402


class Reproj(nn.Module):
    def __init__(self, K, C, P):
        super().__init__()
        self.K = ref.Parameter(K)
        self.C = ref.Parameter(C)
        self.P = ref.Parameter(P)

    def forward(self, observe, cidx, pidx):
        return Reproj.project(self.K[cidx], self.C[cidx], self.P[pidx]) - observe

    @staticmethod
    def project(K, C, P):
        cp = C.Act(P)
        n = -cp[..., :2] / cp[..., [2]]
        radius = n.square().sum(dim=-1, keepdim=True)
        focal, k1, k2 = K[..., :1], K[..., 1:2], K[..., 2:3]
        return focal * (1 + k1 * radius + k2 * radius.square()) * n


CASES = {
    # name: (seed, strategy, steps, start perturbation scale)
    "constant": (0, "constant", 6, 1.0),
    "trustregion": (1, "trustregion", 6, 1.0),
    "reject": (2, "trustregion", 6, 8.0),
}


def strategy(kind):
    return ref.optim.strategy.Constant(damping=1e-6) if kind == "constant" else ref.optim.strategy.TrustRegion()


def run(seed, kind, steps, scale):
    d = problem(seed, scale=scale)
    K0, T0, P0 = (torch.from_numpy(d[k]) for k in ("K0", "T0", "P0"))
    pix, ci, pi_ = torch.from_numpy(d["pix"]), torch.from_numpy(d["cidx"]), torch.from_numpy(d["pidx"])
    model = Reproj(K0.clone(), ref.SE3(T0.clone()), P0.clone())
    opt = ref.optim.LM(model, strategy=strategy(kind), reject=16)
    loss, Ks, Ts, Ps, rej = [], [], [], [], []
    for _ in range(steps):
        loss.append(float(opt.step(input=(pix, ci, pi_))))
        Ks.append(model.K.detach().numpy().copy())
        Ts.append(model.C.detach().tensor().numpy().copy())
        Ps.append(model.P.detach().numpy().copy())
        rej.append(opt.reject_count)
    out = {k: v for k, v in d.items()}
    out.update(loss=np.array(loss), K=np.stack(Ks), T=np.stack(Ts), P=np.stack(Ps), reject=np.array(rej))
    return out


def main():
    torch.set_default_dtype(torch.float64)
    arrays = {}
    for name, (seed, kind, steps, scale) in CASES.items():
        r = run(seed, kind, steps, scale)
        print(name, "loss", r["loss"], "reject", r["reject"])
        for k, v in r.items():
            arrays[f"{name}/{k}"] = v
    assert arrays["reject/reject"].sum() > 0, "the far start must reject at least one trial"
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
