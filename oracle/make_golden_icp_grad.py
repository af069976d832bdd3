"""Goldens for the gradients of pp.module.ICP from the REFERENCE's own autograd (pypose v0.9.5, fp64, CPU):
    PYPOSE_REFERENCE=<path to the reference checkout> python oracle/make_golden_icp_grad.py   # writes tests/golden/icp_grad.npz

Non-degenerate clouds (full-rank cross-covariances, distinct nearest neighbours), batched and broadcast, with and
without init, ord 1, 2 and inf.  Per case: the inputs, the iteration count, the forward result, and the gradients of
source, target and init for two losses on the returned T: sum W * T.matrix() and sum w . T.Act(probe).  Every rotation
the reference converts (each step and the result) is asserted to take mat2SE3's w >= 0 branch, where its quaternion
sign rule and pp.module.ICP's agree.
"""
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "icp_grad.npz")
torch.set_default_dtype(torch.float64)


def rand_se3(shape, sigma, gen):
    return ref.se3(sigma * torch.randn(*shape, 6, generator=gen)).Exp()


def cloud(shape, gen):
    return torch.rand(*shape, 3, generator=gen) * 2 - 1


def cases(gen):
    out = []
    for ordv, tag in ((2, "o2"), (1, "o1"), (math.inf, "oinf")):
        src = cloud((3, 60), gen)
        tgt = rand_se3((3, 1), 0.08, gen).Act(src) + 0.01 * torch.randn(3, 60, 3, generator=gen)
        out.append((f"batched_{tag}", src, tgt, None, ordv))
    src = cloud((3, 50), gen)
    tgt = rand_se3((3, 1), 0.08, gen).Act(src)[:, :45] + 0.01 * torch.randn(3, 45, 3, generator=gen)
    out.append(("batched_init_o2", src, tgt, rand_se3((3,), 0.03, gen), 2))
    one = cloud((1, 55), gen)
    out.append(("bcast_src_o2", one, rand_se3((2, 1), 0.08, gen).Act(one) + 0.01 * torch.randn(2, 55, 3, generator=gen),
                None, 2))
    out.append(("bcast_tgt_init_o1", rand_se3((2, 1), 0.08, gen).Act(one) + 0.01 * torch.randn(2, 55, 3, generator=gen),
                one, rand_se3((2,), 0.02, gen), 1))
    src = cloud((2, 40), gen)
    tgt = rand_se3((2, 1), 0.06, gen).Act(src) + 0.01 * torch.randn(2, 40, 3, generator=gen)
    out.append(("bcast_init_oinf", src, tgt, rand_se3((1,), 0.02, gen), math.inf))
    return out


def check_branch(R):
    """mat2SE3 keeps w >= 0 for R (its trace branch, or a non-negative branch formula)."""
    q = ref.mat2SO3(R, check=False).tensor()
    assert bool((q[..., 3] >= 0).all()), "a rotation outside the agreeing branch"


def main():
    gen = torch.Generator().manual_seed(11)
    g = {}
    for name, src, tgt, init, ordv in cases(gen):
        B = torch.broadcast_shapes(src.shape[:-2], tgt.shape[:-2], *([init.shape[:-1]] if init is not None else []))
        W = torch.randn(*B, 4, 4, generator=gen)
        probe = torch.randn(*B, 5, 3, generator=gen)
        w = torch.randn(*B, 5, 3, generator=gen)
        p = f"{name}/"
        g[p + "source"], g[p + "target"], g[p + "ord"] = src.numpy(), tgt.numpy(), -1 if ordv == math.inf else ordv
        if init is not None:
            g[p + "init"] = init.tensor().numpy()
        g[p + "W"], g[p + "probe"], g[p + "w"] = W.numpy(), probe.numpy(), w.numpy()
        for li in range(2):
            s = src.clone().requires_grad_()
            t = tgt.clone().requires_grad_()
            i = ref.SE3(init.tensor().clone()).requires_grad_() if init is not None else None
            st = ref.utils.ReduceToBason(steps=15)
            T = ref.module.ICP(stepper=st)(s, t, ord=ordv, init=i)
            check_branch(T.matrix()[..., :3, :3])
            L = (T.matrix() * W).sum() if li == 0 else (T.unsqueeze(-2).Act(probe) * w).sum()
            L.backward()
            g[p + "steps"], g[p + "result"] = st.steps, T.detach().tensor().numpy()
            g[p + f"gsrc{li}"], g[p + f"gtgt{li}"] = s.grad.numpy(), t.grad.numpy()
            if init is not None:
                g[p + f"ginit{li}"] = i.grad.numpy()
        # every step's rotation, re-run with the recorded count (the reference does not expose them)
        temporal = src if init is None else init.unsqueeze(-2).Act(src)
        tg = tgt.expand(B + tgt.shape[-2:])
        for _ in range(int(g[p + "steps"])):
            idx = ref.knn(temporal, tg, k=1, ord=ordv, dim=-1)[1]
            idx = idx.expand(B + src.shape[-2:-1] + (1,))
            T = ref.svdtf(temporal, torch.gather(tg, -2, idx.expand(B + src.shape[-2:])))
            check_branch(T.matrix()[..., :3, :3])
            temporal = T.unsqueeze(-2) @ temporal
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, len(g))


if __name__ == "__main__":
    main()
