"""Goldens for pp.svdstf, pp.nbr_filter, pp.random_filter, pp.voxel_filter and pp.knn_filter from the REFERENCE (pypose
v0.9.5, CPU):
    PYPOSE_REFERENCE=<path to the reference checkout> python oracle/make_golden_pcfilter.py   # writes tests/golden/pcfilter.npz

Every case of the reference's tests/function/test_downsample.py is stored as data, plus seeded cases.  knn_filter with a
radius is stored only where the reference is right (its kept rows are the cloud's first rows and every selected
neighbour index is below their number); neighbour sets have no ties at the k-th place.
"""
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "pcfilter.npz")

DOC6 = [[0., 0., 0.], [1., 0., 0.], [0., 1., 0.], [0., 1., 1.], [10., 1., 1.], [10., 1., 10.]]
ROWS5 = [[1., 2.], [4., 5.], [7., 8.], [10., 11.], [13., 14.]]


def voxel_cases(g):
    gen = torch.Generator().manual_seed(11)
    cases = [
        ("t_2d", torch.tensor(ROWS5), [5., 5.]),
        ("t_doc", torch.tensor(DOC6), [1., 1., 1.]),
        ("t_doc4", torch.cat([torch.tensor(DOC6), torch.zeros(6, 1)], 1), [1., 1., 1.]),
        ("t_4col", torch.cat([torch.tensor(ROWS5), torch.zeros(5, 2)], 1), [5., 5., 1, 1]),
        ("t_vdim1", torch.tensor(ROWS5), [5.]),
        ("t_docstring", torch.tensor([[1., 2., 3.], [4., 5., 6.], [7., 8., 9.], [10., 11., 12.], [13., 14., 15.]]),
         [5., 5., 5.]),
    ]
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        cases.append((f"rand_{tag}", (torch.rand(4000, 3, generator=gen, dtype=torch.float64) * 4 - 2).to(dt),
                      [0.5, 0.6, 0.45]))
        cases.append((f"vdim_lt_d_{tag}", torch.randn(1500, 5, generator=gen, dtype=torch.float64).to(dt), [0.4, 0.3, 0.5]))
        cases.append((f"vdim1_{tag}", torch.randn(1000, 3, generator=gen, dtype=torch.float64).to(dt), [0.05]))
        cases.append((f"negative_{tag}", torch.randn(1500, 3, generator=gen, dtype=torch.float64).to(dt), [-0.2, 0.3, -0.25]))
        cases.append((f"one_voxel_{tag}", (torch.rand(700, 4, generator=gen, dtype=torch.float64) * 0.5).to(dt), [1.0, 1.0]))
    cases.append(("v01_f64", torch.rand(2000, 3, generator=gen, dtype=torch.float64) * 3, [0.1, 0.1, 0.1]))
    for name, pts, vox in cases:
        out = ref.voxel_filter(pts, vox)
        g[f"voxel/{name}/points"], g[f"voxel/{name}/voxel"] = pts.numpy(), np.array(vox, np.float64)
        g[f"voxel/{name}/out"] = out.numpy()


def nbr_cases(g):
    pts = torch.tensor(DOC6)
    for name, kw in (("t_r5", dict(nbr=2, radius=5)), ("t_r12", dict(nbr=2, radius=12)),
                     ("t_r10_p2", dict(nbr=2, radius=10, pdim=2)), ("t_r10_p3", dict(nbr=2, radius=10, pdim=3))):
        _, mask = ref.nbr_filter(pts, return_mask=True, **kw)
        g[f"nbr/{name}/points"], g[f"nbr/{name}/mask"] = pts.numpy(), mask.numpy()
        g[f"nbr/{name}/args"] = np.array([kw["nbr"], kw["radius"], kw.get("pdim", 0), 2], np.float64)
    gen = torch.Generator().manual_seed(12)
    lattice = [("lat_r1", 3, dict(nbr=3, radius=1.0)), ("lat_r15", 3, dict(nbr=6, radius=1.5)),
               ("lat_r2_ord1", 3, dict(nbr=4, radius=2.0, ord=1)), ("lat_r1_ordinf", 3, dict(nbr=8, radius=1.0, ord=math.inf)),
               ("lat_p2", 4, dict(nbr=5, radius=1.0, pdim=2)), ("lat_d5", 5, dict(nbr=2, radius=1.0))]
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        for name, D, kw in lattice:
            pts = torch.randint(0, 7, (600, D), generator=gen).to(dt)          # integer lattice: exact distances
            _, mask = ref.nbr_filter(pts, return_mask=True, **kw)
            key = f"nbr/{name}_{tag}/"
            g[key + "points"], g[key + "mask"] = pts.numpy(), mask.numpy()
            o = kw.get("ord", 2)
            g[key + "args"] = np.array([kw["nbr"], kw["radius"], kw.get("pdim", 0), -1 if o == math.inf else o], np.float64)


def knn_cases(g):
    p1 = torch.tensor(DOC6)
    p2 = torch.tensor([[1., 0., 0.], [1., 0., 0.], [0., 1., 0.], [4., 1., 1.], [10., 1., 1.], [1., 1., 10.]])
    cases = [("t_p1", p1, dict(k=2)), ("t_p2", p2, dict(k=2)), ("t_batch", torch.stack([p1, p2]), dict(k=2)),
             ("t_doc_radius", p1, dict(k=2, radius=5))]
    gen = torch.Generator().manual_seed(13)
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        x = torch.randn(2, 3, 40, 4, generator=gen, dtype=torch.float64).to(dt)
        cases += [(f"batch_{tag}", x, dict(k=3, pdim=3)), (f"batch_ord1_{tag}", x, dict(k=5, ord=1)),
                  (f"batch_ordinf_{tag}", x[0], dict(k=4, ord=math.inf, pdim=2))]
        # clusters first, outliers last: the kept rows are the cloud's first rows
        c = torch.randn(80, 3, generator=gen, dtype=torch.float64) * 0.2
        far = torch.randn(6, 3, generator=gen, dtype=torch.float64) * 3 + 10 * torch.sign(torch.randn(6, 3, generator=gen, dtype=torch.float64))
        cases.append((f"radius_{tag}", torch.cat([c, far]).to(dt), dict(k=3, radius=1.0)))
    for name, pts, kw in cases:
        out = ref.knn_filter(pts, **kw)
        if "radius" in kw:                  # only where the reference is right: compare with the full-cloud gather
            d = torch.linalg.norm(pts[..., None, :, :] - pts[..., :, None, :], dim=-1, ord=kw.get("ord", 2))
            keep = (d <= kw["radius"]).sum(-1) - 1 >= kw["k"]
            idx = d[keep].topk(kw["k"] + 1, largest=False).indices
            assert keep[:int(keep.sum())].all() and int(idx.max()) < int(keep.sum()), name
            assert torch.equal(out, pts[idx].mean(-2)), name
        g[f"knnf/{name}/points"], g[f"knnf/{name}/out"] = pts.numpy(), out.numpy()
        o = kw.get("ord", 2)
        g[f"knnf/{name}/args"] = np.array([kw["k"], kw.get("pdim", 0), kw.get("radius", -1.0), -1 if o == math.inf else o])


def svdstf_cases(g):
    src = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0., 1., 0.]])
    tgt = torch.tensor([[1., 1., 1.], [2., 1., 1.], [1., 2., 1.]])
    gen = torch.Generator().manual_seed(14)
    s = torch.randn(4, 50, 3, generator=gen, dtype=torch.float64)
    T = ref.Sim3(torch.cat([torch.randn(4, 3, generator=gen, dtype=torch.float64),
                            ref.randn_SO3(4, sigma=0.5, dtype=torch.float64).tensor(),
                            torch.rand(4, 1, generator=gen, dtype=torch.float64) + 0.5], -1))
    t = T.unsqueeze(-2).Act(s) + 0.01 * torch.randn(4, 50, 3, generator=gen, dtype=torch.float64)
    for name, a, b, ws in (("doc", src, tgt, True), ("noisy", s, t, True), ("noscale", s, t, False)):
        out = ref.svdstf(a, b, with_scale=ws)
        g[f"svdstf/{name}/source"], g[f"svdstf/{name}/target"] = a.numpy(), b.numpy()
        g[f"svdstf/{name}/with_scale"], g[f"svdstf/{name}/out"] = int(ws), out.tensor().numpy()
        g[f"svdstf/{name}/matrix"] = out.matrix()[..., :3, :].numpy()


def random_cases(g):
    g["random/shapes"] = np.array([[5, 10, 5, 3], [5, 10, 5, 2]])      # B, N, num, D of test_random


def main():
    torch.manual_seed(0)
    g = {}
    voxel_cases(g)
    nbr_cases(g)
    knn_cases(g)
    svdstf_cases(g)
    random_cases(g)
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, len(g), os.path.getsize(OUT))


if __name__ == "__main__":
    main()
