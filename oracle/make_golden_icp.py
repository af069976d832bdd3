"""Goldens for pp.knn, pp.module.ICP and pp.utils.ReduceToBason from the REFERENCE (pypose v0.9.5, CPU):
    PYPOSE_REFERENCE=<path to the reference checkout> python oracle/make_golden_icp.py   # writes tests/golden/icp.npz
"""
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "icp.npz")


class Recorder(ref.utils.ReduceToBason):
    """The reference stepper, keeping the loss of every step and the state after it."""

    def reset(self):
        super().reset()
        self.trace = []

    def step(self, loss):
        super().step(loss)
        self.trace.append((loss.clone() if torch.is_tensor(loss) else loss, self.steps, self.patience_count, self._continual))


def knn_cases(g):
    gen = torch.Generator().manual_seed(5)
    cases = [
        ("k1_ord2", (2, 37, 3), (2, 50, 3), dict(k=1, ord=2)),
        ("k4_ord2", (2, 37, 3), (2, 50, 3), dict(k=4, ord=2)),
        ("k3_ord1_largest", (3, 20, 3), (3, 41, 3), dict(k=3, ord=1, largest=True)),
        ("k5_ordinf", (2, 33, 3), (2, 29, 3), dict(k=5, ord=math.inf)),
        ("bcast_ref", (1, 25, 3), (4, 30, 3), dict(k=2, ord=2)),
        ("bcast_nbr", (2, 3, 25, 2), (1, 40, 2), dict(k=6, ord=2)),
        ("d5_k8", (2, 19, 5), (2, 64, 5), dict(k=8, ord=2)),
        ("dups_k5", (2, 31, 3), (2, 40, 3), dict(k=5, ord=2)),
    ]
    for name, rs, ns, kw in cases:
        r = torch.randn(*rs, dtype=torch.float64, generator=gen)
        n = torch.randn(*ns, dtype=torch.float64, generator=gen)
        if name.startswith("dups"):
            n[..., 20:40, :] = n[..., 0:20, :]             # every neighbour twice
            r[..., :5, :] = n[..., 3:8, :]                 # queries on top of duplicated neighbours
        out = ref.knn(r, n, **kw)
        g[f"knn/{name}/ref"], g[f"knn/{name}/nbr"] = r.numpy(), n.numpy()
        g[f"knn/{name}/k"], g[f"knn/{name}/ord"] = kw["k"], kw["ord"] if kw["ord"] != math.inf else -1
        g[f"knn/{name}/largest"] = int(kw.get("largest", False))
        g[f"knn/{name}/values"], g[f"knn/{name}/indices"] = out.values.numpy(), out.indices.numpy()


def l_wall(n_points, gen, dtype):
    """The L-shaped planar wall and the noisy arc of the reference's batched ICP test."""
    x1, y1 = torch.linspace(0, 10, n_points // 2), torch.zeros(n_points // 2)
    x2, y2 = torch.full((n_points // 2,), 10.0), torch.linspace(20, 0, n_points // 2)
    wall = torch.stack((torch.cat((x1, x2)), torch.cat((y1, y2)), torch.zeros(n_points)), 1)
    th = torch.linspace(0, 0.5 * 3.14159265, n_points)
    arc = torch.stack((10 + 10 * torch.cos(th) + torch.randn(n_points, generator=gen),
                       20 - 10 * torch.sin(th) + torch.randn(n_points, generator=gen),
                       torch.randn(n_points, generator=gen)), 1)
    src = torch.stack((wall, arc), 0).to(dtype)
    v = torch.tensor([[-0.5, -0.3, 0.02, 0, 0, 0.0499792, 0.9987503],
                      [-0.2, 0.1, 0.1, 0.1304815, 0.0034168, -0.025953, 0.9911051]], dtype=torch.float64)
    v[:, 3:] /= v[:, 3:].norm(dim=-1, keepdim=True)
    tf = ref.SE3(v.to(dtype))
    return src, tf.unsqueeze(-2).Act(src)


def rand_se3(n, sigma, gen):
    return ref.se3(sigma * torch.randn(n, 6, generator=gen, dtype=torch.float64)).Exp()


def icp_cases(g):
    gen = torch.Generator().manual_seed(9)
    scenes = []
    for dt, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        cloud = (torch.rand(3, 300, 3, generator=gen, dtype=torch.float64) * 2 - 1).to(dt)
        tf = rand_se3(3, 0.1, gen).to(dt)
        tgt = tf.unsqueeze(-2).Act(cloud) + 0.01 * torch.randn(3, 300, 3, generator=gen, dtype=torch.float64).to(dt)
        scenes.append((f"rand_{tag}", cloud, tgt, None, {}))
        big = (torch.rand(2, 350, 3, generator=gen, dtype=torch.float64) * 2 - 1).to(dt)
        tf2 = rand_se3(2, 0.05, gen).to(dt)
        scenes.append((f"unequal_{tag}", tf2.unsqueeze(-2).Act(big[:, :200]), big, None, {}))
        one = (torch.rand(1, 250, 3, generator=gen, dtype=torch.float64) * 2 - 1).to(dt)
        tf3 = rand_se3(2, 0.08, gen).to(dt)
        scenes.append((f"bcast_src_{tag}", one, tf3.unsqueeze(-2).Act(one), None, {}))
        scenes.append((f"bcast_tgt_{tag}", tf3.unsqueeze(-2).Act(one), one, None, dict(patience=3, steps=100)))
        init = rand_se3(3, 0.05, gen).to(dt)
        scenes.append((f"init_{tag}", cloud, tgt, init, dict(ord=1)))
        src, tgtw = l_wall(400, gen, dt)
        scenes.append((f"lwall_{tag}", src, tgtw, None, {}))
    for name, src, tgt, init, kw in scenes:
        ordv = kw.pop("ord", 2)
        st = Recorder(**{"steps": 200, **kw})
        icp = ref.module.ICP(stepper=st)
        out = icp(src, tgt, ord=ordv, init=init)
        g[f"icp/{name}/source"], g[f"icp/{name}/target"] = src.numpy(), tgt.numpy()
        if init is not None:
            g[f"icp/{name}/init"] = init.tensor().numpy()
        g[f"icp/{name}/ord"] = ordv
        g[f"icp/{name}/steps_max"] = st.max_steps
        g[f"icp/{name}/patience"] = st.patience
        g[f"icp/{name}/result"] = out.tensor().numpy()
        g[f"icp/{name}/losses"] = torch.stack([t[0] for t in st.trace]).numpy()
        g[f"icp/{name}/steps"] = st.steps


def stepper_cases(g):
    seqs = {
        "tol": ([1.0, 0.5, 0.1, 1e-6], {}),
        "maxsteps": ([1.0 / (i + 1) for i in range(12)], dict(steps=7)),
        "patience": ([1.0, 0.9, 0.8999, 0.89985, 0.8998, 0.89979, 0.89978, 0.8997, 0.5], dict(patience=3)),
        "zero": ([1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0], dict(patience=2, tol=-1.0)),
        "batched": ([[1.0, 2.0], [0.5, 1e-6], [0.4999, 1e-6], [0.49985, 1e-7], [1e-6, 1e-7]], dict(patience=2)),
        "batched_f32": ([[1.0, 2.0], [0.99995, 1.9999], [0.9999, 1.99985], [0.99988, 1.9998], [0.5, 0.5]], dict(patience=2)),
    }
    for name, (losses, kw) in seqs.items():
        dt = torch.float32 if name.endswith("f32") else torch.float64
        st = ref.utils.ReduceToBason(**{"steps": 100, **kw})
        trace = []
        for l in losses:
            if not st.continual():
                break
            st.step(torch.tensor(l, dtype=dt))
            trace.append((st.steps, st.patience_count, int(st._continual)))
        g[f"stepper/{name}/losses"] = np.array(losses, dtype=np.float32 if dt == torch.float32 else np.float64)
        g[f"stepper/{name}/kw"] = np.array([kw.get("steps", 100), kw.get("patience", 5), kw.get("decreasing", 1e-3),
                                            kw.get("tol", 1e-5)])
        g[f"stepper/{name}/trace"] = np.array(trace)


def main():
    g = {}
    knn_cases(g)
    icp_cases(g)
    stepper_cases(g)
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, len(g))


if __name__ == "__main__":
    main()
