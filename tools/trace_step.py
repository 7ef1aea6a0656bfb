"""Kernel timeline of the CUDA-graph-replayed hot step (CUPTI via torch.profiler): true in-graph
durations, stream overlap and gaps.  Usage (on the GPU): python tools/trace_step.py [config]"""
import collections, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import ProfilerActivity, profile
import bench

name = sys.argv[1] if len(sys.argv) > 1 else "baby"
dev = torch.device("cuda")
from mmssl_b200.hotstep import HotStepConfig
from mmssl_b200.synthetic import CONFIGS
U, I, nnz, d, K, dv, dt = CONFIGS[name]
ds, P, feats, graphs, _ = bench.build_problem(name, 2022, dev)
tr = bench.HotStepTrainer(P, feats, graphs, HotStepConfig(embed_size=d, n_layers=K, batch_size=1024), 1024)
for _ in range(5):
    tr.hs.replay()
torch.cuda.synchronize()
N = 5
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(N):
        tr.hs.replay()
    torch.cuda.synchronize()
evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.name not in ("cudaGraphLaunch",)]
ks = sorted(((e.time_range.start, e.time_range.end, e.name, getattr(e, "stream", None)) for e in evs), key=lambda t: t[0])
print("cuda events:", len(ks))
# split into replays by the adamw kernel
steps, cur = [], []
for k in ks:
    cur.append(k)
    if "adamw_kernel" in k[2]:
        steps.append(cur); cur = []
last = steps[-1]
t0 = last[0][0]
span = last[-1][1] - t0
busy = sum(e - s for s, e, _, _ in last)
print(f"step span {span:.1f} us, sum of kernel durations {busy:.1f} us, kernels {len(last)}")
agg = collections.OrderedDict()
for s, e, n, st in last:
    n = n.replace("void ", "").replace("mmssl::", "").split("(")[0][:58]
    agg.setdefault(n, [0, 0.0]); agg[n][0] += 1; agg[n][1] += e - s
for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{t:8.1f} us x{c:3d}  {n}")
print("--- timeline (start_us, dur_us, stream, name)")
for s, e, n, st in last:
    print(f"{s - t0:8.1f} {e - s:7.1f}  s{st}  {n.replace('void ', '').replace('mmssl::', '').split('(')[0][:70]}")
