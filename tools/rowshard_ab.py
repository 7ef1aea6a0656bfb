"""One problem, the row-sharded whole hot step with ONE and with TWO streams (the modality branch beside the id / GCN branch,
each with its own exchange barriers), same process, CUDA graph, CUDA-event timing, max over ranks.  One JSON line per variant
(rank 0), also appended to out/<tag>.jsonl as soon as it exists.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/rowshard_ab.py syn1m [sports] [--steps K] [--tag T]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402
from mmssl_b200.hotstep import HotStepConfig  # noqa: E402
from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem  # noqa: E402
from mmssl_b200.synthetic import TripleSampler  # noqa: E402

names = [a for a in sys.argv[1:] if not a.startswith("--") and not a.isdigit() and a not in ("ab",)] or ["sports"]
steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 20
tag = sys.argv[sys.argv.index("--tag") + 1] if "--tag" in sys.argv else "ab"
names = [n for n in names if n != tag and not n.isdigit()]
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
B = bench.BATCH
for name in names:
    ds, P_cpu, feats_cpu, _, _ = bench.build_problem(name, 2022, None)
    cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=B)
    Pl, fl, gl, pu, pi = shard_problem(P_cpu, feats_cpu, ds.ui_norm, ds.iu_norm, rank, world, dev)
    smp = TripleSampler(ds.train, seed=2022)
    batches = [tuple(torch.from_numpy(x).to(dev) for x in smp.sample(B)) for _ in range(4)]
    g = torch.Generator().manual_seed(7)
    full_masks = tuple(((torch.rand(ds.n_items, ds.embed_size, generator=g) >= cfg.drop_rate) / (1 - cfg.drop_rate)).float() for _ in range(2))
    for streams in ("0", "1"):
        os.environ["MMSSL_ROWSHARD_STREAMS"] = streams
        P = {k: v.clone() for k, v in Pl.items()}
        sh = RowShardedHotStep(P, fl, gl, cfg, B, pu, pi, rank, exchange="multicast", schedule="reduce_scatter")
        sh.masks = tuple(pi.local(m, rank).to(dev) for m in full_masks)
        sh.set_indices(*batches[0])
        sh.capture()
        for s in range(3):
            sh.set_indices(*batches[s % 4]); sh.replay()
        torch.cuda.synchronize()
        dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for s in range(steps):
            sh.set_indices(*batches[s % 4]); sh.replay()
        b.record()
        torch.cuda.synchronize()
        ms = torch.tensor([a.elapsed_time(b) / steps], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        if rank == 0:
            line = json.dumps({"config": name, "n_gpus": world, "streams": 2 if streams == "1" else 1, "ms_per_step": round(float(ms), 4),
                               "schedule": sh.schedule, "steps": steps})
            print(line, flush=True)
            os.makedirs(os.path.join(ROOT, "out"), exist_ok=True)
            with open(os.path.join(ROOT, "out", tag + ".jsonl"), "a") as f:
                f.write(line + "\n")
        del sh, P
        torch.cuda.empty_cache()
dist.destroy_process_group()
