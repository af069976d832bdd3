"""Dev tool: time individual C-ABI Lie kernels on a ring of buffers (CUDA graph, events).
usage: python tools/ab_stream.py [sym ...]   env: B200POSE_STREAM, B200POSE_CTAS_PER_SM, B200POSE_PDL
       python tools/ab_stream.py --chain     bench.py's step with Log's input warm vs cold in L2
       python tools/ab_stream.py --boundary  cost of one launch boundary (Exp and Log, 8 x N rows in 1 vs 8 launches)
       python tools/ab_stream.py --ab VAR=VALUE [runs]   --chain and --boundary with and without one switch, alternated

--ab runs `--chain` and `--boundary` in child processes (the shell reads its switches once per process), alternating
the environment as given (A) with VAR=VALUE added to it (B): A B A B ..., `runs` (default 3) of each, every child waited
for.  It prints, per side, median and spread over the runs of: one 8e6-row launch of Exp and of Log (steady-state
streaming, Log's input cold), one launch boundary of each, the chained step with Log's input warm and cold and the L2
saving; and the card, its power limit and the SM clock sampled under load in each child.

--chain times, on bench.py's ring of 8 batches of 1e6 fp32 elements, Exp(slot j) -> Log(slot j) (the benchmark's
step: Log reads the SE3 batch Exp has just written) and Exp(slot j) -> Log(slot j+4) (same kernels and bytes, but Log's
input was written four steps, 416 MB of traffic, earlier and is no longer in L2).  cold - chained is what L2 reuse
between the two launches saves."""
import ctypes, os, subprocess, sys, json
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pypose_b200 import _C
from pypose_b200._optable import lie_symbols

N = int(os.environ.get("AB_N", 1_000_000))
dev = torch.device("cuda")


def graph_of(calls):
    """warm the calls up once, then capture them into one CUDA graph on a side stream"""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        sp = ctypes.c_void_p(side.cuda_stream)
        for c in calls: c(sp)
        side.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            spc = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            for c in calls: c(spc)
    torch.cuda.synchronize()
    g.replay(); torch.cuda.synchronize()
    return g


def us_per_call(g, calls_per_replay, trips):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(trips): g.replay()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (trips * calls_per_replay)


def run_syms(syms):
    tab = {s: (ct, ins, outs) for s, ct, ins, outs, _ in lie_symbols()}
    res = {}
    for sym in syms:
        ct, ins, outs = tab[sym]
        dt = torch.float32 if ct == "float" else torch.float64
        per = sum(w for _, w in ins + outs) * N * (4 if ct == "float" else 8)
        ring = max(2, int(600e6 // per) + 1)
        f = _C.fn(sym)
        bufs = [([torch.randn(N, w, dtype=dt, device=dev) * 0.5 for _, w in ins],
                 [torch.empty(N, w, dtype=dt, device=dev) for _, w in outs]) for _ in range(ring)]

        def call(j):
            def c(sp):
                i_t, o_t = bufs[j]
                rc = f(*[ctypes.c_void_p(t.data_ptr()) for t in i_t + o_t], N, sp)
                assert rc == 0, rc
            return c
        g = graph_of([call(j) for j in range(ring)])
        us = us_per_call(g, ring, max(1, 4000 // ring))
        res[sym] = {"us": round(us, 2), "GBs": round(per / us / 1e3, 1)}
    return res


def run_chain(regions=5, steps=4000):
    ring = 8                                     # as bench.py: 8 x 76 MB of distinct buffers
    xs = [torch.randn(N, 6, device=dev) * 0.5 for _ in range(ring)]
    Xs = [torch.empty(N, 7, device=dev) for _ in range(ring)]
    ys = [torch.empty(N, 6, device=dev) for _ in range(ring)]
    f_exp, f_log = _C.fn("b200_se3_exp_fwd_f32"), _C.fn("b200_SE3_log_fwd_f32")
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())

    def step(j, k):                              # Exp into slot j, then Log of slot k
        def c(sp):
            _C.check(f_exp(ptr(xs[j]), ptr(Xs[j]), N, sp), "exp")
            _C.check(f_log(ptr(Xs[k]), ptr(ys[k]), N, sp), "log")
        return c
    g_chain = graph_of([step(j, j) for j in range(ring)])
    g_cold = graph_of([step(j, (j + 4) % ring) for j in range(ring)])
    trips = max(1, steps // ring)
    chain, cold = [], []
    for _ in range(regions):                     # alternate the two so drifting clocks hit both alike
        chain.append(us_per_call(g_chain, ring, trips))
        cold.append(us_per_call(g_cold, ring, trips))
    med = lambda v: sorted(v)[len(v) // 2]
    return {"chained_us": round(med(chain), 2), "cold_us": round(med(cold), 2),
            "l2_saving_us": round(med(cold) - med(chain), 2),
            "chained_all": [round(v, 2) for v in chain], "cold_all": [round(v, 2) for v in cold]}


def run_boundary(parts=8, regions=5, trips=200):
    """Cost of one launch boundary: the same 8 x N rows moved by one launch and by 8 launches of N rows over the 8
    slices of the same buffer (one CUDA graph each); (eight - one) / 7 is what each boundary adds."""
    med = lambda v: sorted(v)[len(v) // 2]
    res = {}
    for name, sym, wi, wo in (("exp", "b200_se3_exp_fwd_f32", 6, 7), ("log", "b200_SE3_log_fwd_f32", 7, 6)):
        f = _C.fn(sym)
        x = torch.randn(parts * N, 6, device=dev) * 0.5
        if name == "log":                        # Log of valid SE3 rows
            X = torch.empty(parts * N, 7, device=dev)
            _C.check(_C.fn("b200_se3_exp_fwd_f32")(x.data_ptr(), X.data_ptr(), parts * N, None), "exp")
            x = X
        y = torch.empty(parts * N, wo, device=dev)
        call = lambda k, n: (lambda sp: _C.check(f(x.data_ptr() + k * N * wi * 4, y.data_ptr() + k * N * wo * 4, n, sp), sym))
        g_one = graph_of([call(0, parts * N)])
        g_many = graph_of([call(k, N) for k in range(parts)])
        one, many = [], []
        for _ in range(regions):
            one.append(us_per_call(g_one, 1, trips))
            many.append(us_per_call(g_many, 1, trips))
        res[name] = {"one_launch_us": round(med(one), 2), f"{parts}_launches_us": round(med(many), 2),
                     "per_boundary_us": round((med(many) - med(one)) / (parts - 1), 3),
                     "one_all": [round(v, 2) for v in one], "many_all": [round(v, 2) for v in many]}
        del x, y
    return res


def card_under_load(g):
    """card name, power limit and SM clock, read while replays of graph g keep the GPU busy"""
    for _ in range(3000): g.replay()
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--format=csv,noheader",
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm"], capture_output=True, text=True)
    torch.cuda.synchronize()
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def run_ab(setting, runs=3):
    var, value = setting.split("=", 1)
    sides = {"A": dict(os.environ), "B": {**os.environ, var: value}}
    got = {"A": [], "B": []}
    for _ in range(runs):
        for side in "AB":
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--ab-child"], env=sides[side],
                                 capture_output=True, text=True, check=True).stdout
            got[side].append(json.loads(out.strip().splitlines()[-1]))
    pick = {"exp_one_launch_us": lambda r: r["exp"]["one_launch_us"], "log_one_launch_us": lambda r: r["log"]["one_launch_us"],
            "exp_per_boundary_us": lambda r: r["exp"]["per_boundary_us"], "log_per_boundary_us": lambda r: r["log"]["per_boundary_us"],
            "chained_us": lambda r: r["chained_us"], "cold_us": lambda r: r["cold_us"], "l2_saving_us": lambda r: r["l2_saving_us"]}
    res = {"B": setting, "card": sorted({r["card"] for side in "AB" for r in got[side]})}
    for side in "AB":
        res[side] = {}
        for k, f in pick.items():
            v = sorted(f(r) for r in got[side])
            res[side][k] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    return res


if __name__ == "__main__":
    args = sys.argv[1:]
    if args == ["--chain"]:
        res = run_chain()
    elif args == ["--ab-child"]:
        res = {**run_chain(), **run_boundary()}
        x, X = torch.randn(N, 6, device=dev), torch.empty(N, 7, device=dev)
        res["card"] = card_under_load(graph_of(
            [lambda sp: _C.check(_C.fn("b200_se3_exp_fwd_f32")(x.data_ptr(), X.data_ptr(), N, sp), "exp")]))
    elif args[:1] == ["--ab"] and len(args) in (2, 3):
        res = run_ab(args[1], *map(int, args[2:]))
    elif args == ["--boundary"]:
        res = run_boundary()
    else:
        res = run_syms(args or ["b200_se3_exp_fwd_f32", "b200_SE3_log_fwd_f32"])
    print(json.dumps({"impl": os.environ.get("B200POSE_STREAM", "v2"), "ctas": os.environ.get("B200POSE_CTAS_PER_SM", "half"),
                      "pdl": os.environ.get("B200POSE_PDL", "1"), "n": N, **res}))
