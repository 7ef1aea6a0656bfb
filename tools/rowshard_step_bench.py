"""Row-sharded WHOLE hot step (mmssl_b200/rowshard_step.py, SURVEY 8e) on N GPUs of one box: parity against the single-GPU
fused HotStep on the same problem (`check`) and time per step (CUDA events, max over ranks).  One JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/rowshard_step_bench.py [config] [check] [mc] [graph] [--steps K] [--batch B]     (mc: exchange through the multicast publish kernel instead of NCCL)

Written when round 1 had no GPU time left; the same class runs in tests/test_dist_emu.py with 2 gloo ranks on the CPU emulator."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402
from mmssl_b200.engine import LIVE, P_EI, P_EU  # noqa: E402
from mmssl_b200.hotstep import HotStep, HotStepConfig  # noqa: E402
from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem  # noqa: E402
from mmssl_b200.synthetic import TripleSampler  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
name = args[0] if args and args[0] not in ("check", "mc", "graph", "allgather") else "tiktok"
schedule = "allgather" if "allgather" in args else "reduce_scatter"
check = "check" in args
steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 20
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
B = int(sys.argv[sys.argv.index("--batch") + 1]) if "--batch" in sys.argv else bench.BATCH
ds, P_cpu, feats_cpu, _, _ = bench.build_problem(name, 2022, None)           # the same seeded problem on every rank (host)
cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=B)
Pl, fl, gl, pu, pi = shard_problem(P_cpu, feats_cpu, ds.ui_norm, ds.iu_norm, rank, world, dev)
mode = "multicast" if "mc" in args and world > 1 else "nccl"
sh = RowShardedHotStep(Pl, fl, gl, cfg, B, pu, pi, rank, exchange=mode, schedule=schedule)
smp = TripleSampler(ds.train, seed=2022)
batches = [tuple(torch.from_numpy(x).to(dev) for x in smp.sample(B)) for _ in range(4)]
g = torch.Generator().manual_seed(7)
full_masks = tuple(((torch.rand(ds.n_items, ds.embed_size, generator=g) >= cfg.drop_rate) / (1 - cfg.drop_rate)).float() for _ in range(2))
sh.masks = tuple(pi.local(m, rank).to(dev) for m in full_masks)
res = {"config": name, "n_gpus": world, "scheme": "row-sharded whole hot step", "schedule": sh.schedule, "exchange": ("publish kernel over NVSwitch multicast / peer stores + signal-pad barrier (no NCCL)" if mode == "multicast" else "NCCL all-gather per SpMM operand"), "batch": B}

if check:
    # Parity of ONE step without the optimiser: the five loss terms and every live gradient (table gradients: the rank's rows).
    # Parameters after AdamW are NOT the yardstick: m / (sqrt(v) + eps) turns a 1e-9 difference in a gradient entry of size 1e-8
    # into a full-size (lr) difference of the parameter -- on the earlier hardware gradients agreed to 5e-6 where the parameters
    # after two AdamW steps differed by 1e-2 (summation orders differ between the two schemes).  A loose bound on the parameters is kept.
    _, Pd, feats, graphs, _ = bench.build_problem(name, 2022, dev)
    hs = HotStep(Pd, feats, graphs, cfg, batch=B, optimizer_step=False)
    hs.masks = tuple(m.to(dev) for m in full_masks)
    sh.optimizer_step = False
    err, worst = 0.0, ""
    for s in range(2):
        hs.set_indices(*batches[s]); sh.set_indices(*batches[s])
        want, got = hs.run().clone(), sh.run().clone()
        e = float(((got - want).abs() / want.abs().clamp_min(1e-12)).max())
        if e > err:
            err, worst = e, f"losses(step {s})"
        for k in LIVE:
            part = pu if k == P_EU else pi if k == P_EI else None
            a = sh.grads[k] if part is None else sh.grads[k][:part.bounds(rank)[1] - part.bounds(rank)[0]]
            b = hs.grads[k] if part is None else hs.grads[k][part.bounds(rank)[0]:part.bounds(rank)[1]]
            e = float((a - b).abs().max() / hs.grads[k].abs().max().clamp_min(1e-30))
            if e > err:
                err, worst = e, k
    e = torch.tensor([err], device=dev)
    if world > 1:
        dist.all_reduce(e, op=dist.ReduceOp.MAX)
    res["max_rel_err_vs_1gpu"] = float(e)
    res["worst_on_rank0"] = worst
    res["compared"] = "5 loss terms + 7 live gradients of two steps (no optimiser)"
    sh.optimizer_step = True
    del hs, Pd, feats, graphs

use_graph = "graph" in args
if use_graph:
    sh.set_indices(*batches[0])
    sh.capture()
step = sh.replay if use_graph else sh.run
for s in range(3):
    sh.set_indices(*batches[s % 4]); step()
torch.cuda.synchronize()
if world > 1:
    dist.barrier()
sh.n_gathers = sh.gathered_bytes = sh.n_reduce_scatters = 0
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for s in range(steps):
    sh.set_indices(*batches[s % 4]); step()
b.record()
torch.cuda.synchronize()
ms = torch.tensor([a.elapsed_time(b) / steps], device=dev)
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
res.update(ms_per_step=round(float(ms), 4), triples_per_s=round(B / float(ms) * 1e3, 1), gathers_per_step=sh.n_gathers // steps, reduce_scatters_per_step=sh.n_reduce_scatters // steps,
           gathered_MB_per_rank_per_step=round(sh.gathered_bytes / steps / 1e6, 2), graph_capture=use_graph)
if rank == 0:
    print(json.dumps(res))
if world > 1:
    dist.destroy_process_group()
