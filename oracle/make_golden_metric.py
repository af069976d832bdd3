"""Goldens for pp.metric.ape / rpe from the REFERENCE (pypose v0.9.5, CPU):
    PYPOSE_REFERENCE=<path to the reference checkout> python oracle/make_golden_metric.py   # writes tests/golden/metric.npz

Each case stores a recipe for each input array (oracle/metric_oracle.py `synth`: integer hashing and elementwise fp64, so
every machine rebuilds the same bits; the docstring example and two small stamp arrays are stored as values under in/),
the keyword arguments, the reference's statistics, whether it warned and, captured from inside the reference's own calls,
its association indices and pair indices (first differences, int32) and, up to ERR_MAX pairs, its per-pair error
vector.  Each distinct index or error array is stored once, under arr/; the per-case entries are one JSON document,
`cases`, that holds their keys.  The `nposes` cases are
stored from oracle/metric_oracle.py instead (the reference ignores `nposes`); their `from` entry says so.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.dont_write_bytecode = True
import pypose as ref  # noqa: E402
from pypose.metric import ape_rpe as R  # noqa: E402
from oracle import metric_oracle as O  # noqa: E402

ERR_MAX = 400           # per-pair error vectors are stored up to this length
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "metric.npz")

DOC_RSTAMP = [1311868163.8696999550, 1311868163.8731000423, 1311868163.8763999939]
DOC_RPOSE = [[-0.1357000023, -1.4217000008, 1.4764000177, 0.6452999711, -0.5497999787, 0.3362999856, -0.4101000130],
             [-0.1357000023, -1.4218000174, 1.4764000177, 0.6453999877, -0.5497000217, 0.3361000121, -0.4101999998],
             [-0.1358000040, -1.4219000340, 1.4764000177, 0.6455000043, -0.5498999953, 0.3357999921, -0.4101000130]]
DOC_ESTAMP = [1311868164.3631811142, 1311868164.3990259171, 1311868164.4309399128]
DOC_EPOSE = [[0.0000000000, 0.0000000000, 0.0000000000, 0.0000000000, 0.0000000000, 0.0000000000, 1.0000000000],
             [-0.0005019300, 0.0010138600, -0.0020097860, -0.0020761820, -0.0010706080, -0.0007627490, 0.9999969602],
             [0.0004298200, 0.0019603260, -0.0048985220, -0.0043526068, -0.0036625920, -0.0023494449, 0.9999810457]]


class _Spy:
    """Stands in for `torch` inside the reference module to capture the error vector given to torch.max."""
    def __init__(self):
        self.err = None

    def __getattr__(self, k):
        return getattr(torch, k)

    def max(self, x, *a, **k):
        self.err = x.clone()
        return torch.max(x, *a, **k)


def run_ref(fn, rs, rp, es, ep, kw):
    spy = _Spy()
    cap = {}
    mti, pid = R.matching_time_indices, R.pair_id

    def mti_w(s1, s2, *a):
        i1, i2 = mti(s1.clone(), s2.clone(), *a)
        cap['m1'], cap['m2'] = np.array(i1, np.int64), np.array(i2, np.int64)
        return i1, i2

    def pid_w(*a, **k):
        p = pid(*a, **k)
        cap['src'], cap['tgt'] = np.array(p[0], np.int64), np.array(p[1], np.int64)
        return p

    R.torch, R.matching_time_indices, R.pair_id = spy, mti_w, pid_w
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            out = fn(None if rs is None else rs.clone(), ref.SE3(rp.clone()), None if es is None else es.clone(),
                     ref.SE3(ep.clone()), **kw)
        cap['warned'] = np.array(len(w) > 0)
    finally:
        R.torch, R.matching_time_indices, R.pair_id = torch, mti, pid
    cap['err'] = spy.err.numpy()
    vals = [out[k] for k in O.KEYS] if isinstance(out, dict) else [out]
    cap['stats'] = np.array([float(v) for v in vals])
    return cap


def main():
    store = {"in/doc_rstamp": np.array(DOC_RSTAMP, np.float32), "in/doc_estamp": np.array(DOC_ESTAMP, np.float32),
             "in/doc_rpose": np.array(DOC_RPOSE, np.float32), "in/doc_epose": np.array(DOC_EPOSE, np.float32)}
    cases = []

    def add(name, fn, rs, rp, es, ep, **kw):
        cases.append((name, fn, rs, rp, es, ep, kw))

    def sl(r, *a):
        return ["slice", r] + list(a)

    # docstring example: fp32 stamps, all round to one value, so every pose matches long index 0
    drs, des, drp, dep = (["in", f"in/doc_{k}"] for k in ("rstamp", "estamp", "rpose", "epose"))
    add("doc_ape", "ape", drs, drp, des, dep)
    add("doc_rpe", "rpe", drs, drp, des, dep)
    add("doc_ape_mean", "ape", drs, drp, des, dep, otype='Mean')

    P = ["traj", 1500, 1, False]
    E = ["perturb", P, 2, 0.02]
    rs = ["stamps", 1500, 100.0, 1000.0, 3, 0.002]
    es1 = ["stamps", 500, 30.0, 1000.004, 4, 0.002]
    E3, P3 = sl(E, None, None, 3), sl(P, None, None, 3)
    add("r_longer", "ape", rs, P, es1, E3)
    add("e_longer", "ape", es1, P3, rs, E)
    add("equal_len", "ape", sl(rs, 500), sl(P, 500), es1, sl(E, 500))
    add("offset_pos", "ape", rs, P, es1, E3, offset=0.05, diff=0.02)
    add("offset_neg", "ape", es1, P3, rs, E, offset=-0.05, diff=0.02)
    # duplicate long stamps: ties between equal stamps take the lowest index
    add("dup_long", "ape", ["repeat", ["stamps", 500, 50.0, 5.0, 5, 0.0], 3], P, ["stamps", 400, 40.0, 5.001, 6, 0.01],
        sl(E, 400), diff=0.03)
    # distances exactly equal to diff (binary fractions) are not matches
    store["in/ri"] = np.arange(200, dtype=np.float64) * 0.5
    store["in/ei"] = store["in/ri"][::2] + np.array([0.25, 0.125] * 50)
    add("diff_boundary", "ape", ["in", "in/ri"], sl(P, 200), ["in", "in/ei"], sl(E, 100), diff=0.25)
    add("below_thresh", "ape", sl(rs, 500), sl(P, 500), ["stamps", 300, 30.0, 1004.0, 7, 0.0], sl(E, 300))
    add("none_stamps", "ape", None, sl(P, 800), None, sl(E, 800))
    add("none_stamps_rpe", "rpe", None, sl(P, 800), None, sl(E, 800), delta=2)
    Pm, Em = sl(P, 300), sl(E, 300)
    for et in O.ETYPES:
        for ot in ['All'] + O.KEYS:
            add(f"ape_{et}_{ot}", "ape", None, Pm, None, Em, etype=et, otype=ot)
            add(f"rpe_{et}_{ot}", "rpe", None, Pm, None, Em, etype=et, otype=ot, delta=2)
    # alignment: a rotated, scaled, shifted estimate
    Ea = ["sim3inv", sl(E, 500)]
    for tag, kw in (("align", dict(align=True)), ("scale", dict(scale=True)), ("both", dict(align=True, scale=True)),
                    ("origin", dict(origin=True))):
        add(f"ape_{tag}", "ape", sl(rs, 500), sl(P, 500), es1, Ea, **kw)
        add(f"rpe_{tag}", "rpe", sl(rs, 500), sl(P, 500), es1, Ea, **kw)
    add("rpe_align_dist_all", "rpe", sl(rs, 500), sl(P, 500), es1, Ea, align=True, scale=True,
        associate='distance', delta=0.5, all=True)
    for d in (1, 3):
        for a in (False, True):
            add(f"rpe_frame_d{d}_all{int(a)}", "rpe", rs, P, es1, E3, delta=d, all=a)
    Pp = ["traj", 2000, 8, True]
    Ep = ["perturb", Pp, 9, 0.04]
    for a in (False, True):
        for rp_ in (False, True):
            for rtol in (0.01, 0.1, 0.5):
                add(f"rpe_dist_all{int(a)}_rpair{int(rp_)}_rtol{rtol}", "rpe", None, Pp, None, Ep,
                    associate='distance', delta=0.3, rtol=rtol, all=a, rpair=rp_)
    Pl = ["traj", 5000, 10, True]
    El = ["perturb", Pl, 11, 0.02]
    add("large_ape", "ape", None, Pl, None, El, etype='pose')
    add("large_rpe_dist", "rpe", None, Pl, None, El, associate='distance', delta=1.0, all=True, rpair=True)
    add("large_rpe_walk", "rpe", None, Pl, None, El, associate='distance', delta=1.0)
    add("fp32_poses", "ape", sl(rs, 500), ["f32", sl(P, 500)], es1, ["f32", sl(E, 500)], etype='radian')
    add("fp32_poses_rpe", "rpe", sl(rs, 500), ["f32", sl(P, 500)], es1, ["f32", sl(E, 500)], etype='rotation', delta=3)

    data = dict(store)
    meta = {}
    T = lambda r: None if r is None else torch.from_numpy(O.synth(r, store))   # noqa: E731
    for name, fn, rs_, rp_, es_, ep_, kw in cases:
        cap = run_ref(getattr(ref.metric, fn), T(rs_), T(rp_), T(es_), T(ep_), kw)
        m = _case_meta(fn, rs_, rp_, es_, ep_, kw, "reference")
        for k in ("m1", "m2", "src", "tgt"):        # increasing indices: first differences, shared between cases
            if k in cap:
                m[k] = _shared(data, np.diff(cap[k], prepend=0).astype(np.int32))
        if len(cap['err']) <= ERR_MAX:              # long error vectors: the statistics and the indices pin them
            m["err"] = _shared(data, cap['err'])
        m["stats"] = cap["stats"].tolist()
        m["warned"] = bool(cap["warned"])
        meta[name] = m
    # nposes: the first nposes associated poses (the reference slices coordinates instead); stored from the oracle
    for n_ in (5, 100):
        for fn in ("ape", "rpe"):
            kw = dict(align=True, scale=True, nposes=n_)
            args = (O.synth(sl(rs, 500)), O.synth(sl(P, 500)), O.synth(es1), O.synth(Ea))
            if fn == "ape":
                err, *_ = O.ape(*args, align_=True, scale=True, nposes=n_)
            else:
                err, *_ = O.rpe(*args, align_=True, scale=True, nposes=n_)
            m = _case_meta(fn, sl(rs, 500), sl(P, 500), es1, Ea, kw, "oracle")
            m["stats"] = [float(O.stats(err)[k]) for k in O.KEYS]
            meta[f"nposes{n_}_{fn}"] = m
    data["cases"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, len(meta), "cases")


def _case_meta(fn, rs, rp, es, ep, kw, src):
    m = {"fn": fn, "kw": kw, "from": src}
    for k, v in (("rstamp", rs), ("rpose", rp), ("estamp", es), ("epose", ep)):
        if v is not None:
            m[k] = v
    return m


def _shared(data, a):
    """Store each distinct array once, under arr/<n>; cases hold its key."""
    for k, v in data.items():
        if k.startswith("arr/") and v.dtype == a.dtype and v.shape == a.shape and np.array_equal(v, a):
            return k
    k = f"arr/{sum(1 for k in data if k.startswith('arr/'))}"
    data[k] = a
    return k


if __name__ == "__main__":
    main()
