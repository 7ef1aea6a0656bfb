"""Full training iteration (mmssl_b200/fullstep.py = main.py:333-434: D step + G step + both optimisers + graph rebuilds) on one
GPU, timed with CUDA events, next to the hot step alone and to the oracle's CPU restatement of the same iteration.
SURVEY 8d: "also report full step for C1-C3".  Prints one JSON line.

    python tools/fullstep_bench.py [config=baby] [--steps K] [--warmup W] [--gemm tc|simt|cublas] [--cpu-steps N]

Not part of bench.py's contract (the headline metric is the hot step); H100 numbers in DESIGN section 6."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("config", nargs="?", default="baby")
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--gemm", default=os.environ.get("MMSSL_GAN_GEMM", "simt"), choices=["tc", "simt", "cublas"])
ap.add_argument("--cpu-steps", type=int, default=2)
ap.add_argument("--seed", type=int, default=2022)
ap.add_argument("--batch", type=int, default=0, help="0 = bench.BATCH (1024, the reference default)")
ap.add_argument("--phases", action="store_true", help="CUDA-event breakdown: first forward, 3x u_sim, D step, G step (hot step + generator side)")
a = ap.parse_args()

import bench  # noqa: E402  (problem builder shared with the headline benchmark)
from mmssl_b200 import gan, gan_ops  # noqa: E402
from mmssl_b200.fullstep import FullStep, FullStepConfig  # noqa: E402
from mmssl_b200.hotstep import HotStepConfig  # noqa: E402
from mmssl_b200.synthetic import TripleSampler  # noqa: E402

gan_ops.GEMM_IMPL = a.gemm
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
B = a.batch or bench.BATCH
ds, P, feats, graphs, feats_cpu = bench.build_problem(a.config, a.seed, dev)
U, I, d = ds.n_users, ds.n_items, ds.embed_size
h1, h2 = int(I / 4), int(I / 8)
g = torch.Generator().manual_seed(a.seed + 1)


def d_state(device):
    """Discriminator(n_items) after weights_init (main.py:73, :133-136): kaiming-normal Linear weights, zero biases."""
    kn = lambda o, i: torch.randn(o, i, generator=g) * (2.0 / i) ** 0.5
    s = {"net.0.weight": kn(h1, I), "net.0.bias": torch.zeros(h1), "net.2.weight": torch.ones(h1), "net.2.bias": torch.zeros(h1),
         "net.2.running_mean": torch.zeros(h1), "net.2.running_var": torch.ones(h1), "net.2.num_batches_tracked": torch.zeros((), dtype=torch.int64),
         "net.4.weight": kn(h2, h1), "net.4.bias": torch.zeros(h2), "net.6.weight": torch.ones(h2), "net.6.bias": torch.zeros(h2),
         "net.6.running_mean": torch.zeros(h2), "net.6.running_var": torch.ones(h2), "net.6.num_batches_tracked": torch.zeros((), dtype=torch.int64),
         "net.8.weight": kn(1, h2), "net.8.bias": torch.zeros(1)}
    return {k: v.to(device) for k, v in s.items()}


S_cpu = d_state("cpu")
R = ds.train.tocsr()
R.sort_indices()
t64 = lambda x: torch.from_numpy(np.asarray(x, dtype=np.int64)).to(dev)
cfg = FullStepConfig(hot=HotStepConfig(embed_size=d, n_layers=ds.n_layers, batch_size=B), gan=gan.GanHyper())
fs = FullStep(P, {k: v.clone().to(dev) for k, v in S_cpu.items()}, feats, t64(R.indptr), t64(R.indices), graphs[0], graphs[1], cfg, batch=B)
smp = TripleSampler(ds.train, seed=a.seed)
batches = [tuple(torch.from_numpy(x).to(dev) for x in smp.sample(B)) for _ in range(8)]


def run(n):
    for s in range(n):
        out = fs.step(*batches[s % len(batches)])
    return out


phase_ev = {}
if a.phases:                 # wrap the pieces of FullStep._body with event pairs (eager mode only)
    from mmssl_b200 import fullstep as _F

    def timed(name, fn):
        def w(*x, **k):
            e = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            e[0].record()
            r = fn(*x, **k)
            e[1].record()
            phase_ev.setdefault(name, []).append(e)
            return r
        return w
    fs.hs.engine.forward = timed("forward (each of the 2 per iteration)", fs.hs.engine.forward)
    fs.hs.engine.backward = timed("backward", fs.hs.engine.backward)
    _F.gan.u_sim_forward = timed("u_sim forward (each of the 5)", _F.gan.u_sim_forward)
    _F.gan.u_sim_backward = timed("u_sim backward (each of the 2)", _F.gan.u_sim_backward)
    _F.gan.d_step = timed("D step (3 D calls + penalty sweeps + Adam)", _F.gan.d_step)
    _F.gan.g_side = timed("G side (D call + input gradient)", _F.gan.g_side)
    fs.hs.run = timed("G step total (HotStep.run incl. generator side, backward, AdamW)", fs.hs.run)


run(a.warmup)
torch.cuda.synchronize()
from mmssl_b200 import _lib  # noqa: E402
_lib.launch_count = 0
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
out = run(a.steps)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / a.steps
launches = _lib.launch_count / a.steps
phases = {k: round(sum(e0.elapsed_time(e1) for e0, e1 in v[-a.steps:]) / max(1, len(v[-a.steps:])), 4) for k, v in phase_ev.items()}
res = {"metric": "bpr_triples_per_sec_full_step", "unit": "triples/s", "value": B / ms * 1e3, "ms_per_step": ms, "n_gpus": 1,
       "steps": a.steps, "warmup": a.warmup, "config": {"workload": a.config, "U": U, "I": I, "nnz": int(ds.nnz), "d": d, "batch": B,
                                                          "gan_gemm": a.gemm, "graph_capture": False, "modality_graphs": "empty after iteration 1 (T=1, reference quirk)"},
       "gpu_launches_per_step": launches, "batch_loss": float(out["batch_loss"]), "loss_D": float(out["loss_D"]),
       "big_gemm_gflop_per_step": 11 * 2 * 2 * B * I * h1 / 1e9}
if phases:
    res["phase_ms_per_call"] = phases

if a.cpu_steps > 0:          # the oracle's restatement of the same iteration on the host cores, a bounded sample (bench.py owns that leg)
    res["cpu_baseline"] = bench.cpu_full_step_baseline(a.config, a.seed, a.cpu_steps, B, S_cpu)
print(json.dumps(res))
