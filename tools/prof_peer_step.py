"""Dev: wall clock and kernel durations of the sharded reprojection step (torchrun, one rank per GPU).
python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 tools/prof_peer_step.py [C M]"""
import datetime
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, ".")
import pypose_b200 as pp          # noqa: E402
import bench_legs as BL           # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if os.environ.get("NCCL_DEBUG", "").upper() == "VERSION":
    os.environ["NCCL_DEBUG"] = "WARN"
dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=120))
C, M = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (10_000, 1_000_000)
init, inp = BL._reproj_problem(pp, dev, C, M, rank, world, 77, sorted_split=True)
net = pp.module.PoseReproj(init.clone())
opt = pp.optim.LM(net, strategy=pp.optim.strategy.TrustRegion(), group=True)
for _ in range(20):
    opt.step(inp)
torch.cuda.synchronize(); dist.barrier()
steps = 1000
t0 = time.perf_counter()
for _ in range(steps):
    opt.step(inp)
torch.cuda.synchronize()
dt = (time.perf_counter() - t0) / steps
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(50):
        opt.step(inp)
    torch.cuda.synchronize()
dist.barrier()
if rank == 0:
    print(f"C={C} M={M} world={world}: {dt * 1e6:.1f} us per step (wall clock, converged state)")
    rows = [(e.key, e.device_time_total / max(e.count, 1), e.count) for e in prof.key_averages() if e.device_time_total > 0]
    for key, us, cnt in sorted(rows, key=lambda r: -r[1])[:8]:
        print(f"   {us:9.2f} us x{cnt:4d}  {key[:110]}")
dist.destroy_process_group()
