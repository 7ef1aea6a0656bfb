"""Recommendation throughput (recommend.py, mmssl_recommend_topk): users ranked per second over every user of a synthetic problem
(bench.build_problem: baby / sports / syn1m; exclusion = the training rows of its graph), seeded random fp32 tables.

    python tools/recommend_bench.py [--configs baby,sports,syn1m] [--ks 20,100] [--iters K] [--warmup W]
        one GPU: per config and k, the ranking kernel alone (CUDA events) and the whole chunked export to a temporary directory
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/recommend_bench.py --sharded [config] [--k K]
        the row-sharded path (RowShardedHotStep.final_embeddings + ShardedRecommender): eval-mode forward, item all-gather,
        ranking of the rank's users and the rank's export, timed separately, max over ranks

Reports the algorithmic work 2 * users * items * d FLOP over the ranking kernel's time against the 67 TFLOP/s fp32 CUDA-core
bound of the H100 SXM (the sweep is fp32 FMA).  One JSON line, with the card name and power limit read in the same run.
Not part of bench.py's contract; H100 numbers in DESIGN section 6."""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402
from mmssl_b200 import recommend  # noqa: E402
from mmssl_b200.evaluate import _device_csr  # noqa: E402

FP32_BOUND = 67e12
opt = lambda k, dflt: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else dflt
iters, warmup = int(opt("--iters", 3)), int(opt("--warmup", 1))
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)


def card():
    q = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return dict(card=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip() if q.returncode == 0 else None)


def train_rows(ds):
    tr = ds.train.tocsr()
    tr.sort_indices()
    return tr.indptr.astype(np.int64), tr.indices


def timed(fn):
    """Mean ms of fn over `iters` calls after `warmup`, CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def one_gpu():
    res = {"mode": "one GPU", "iters": iters, "rows": []}
    for name in opt("--configs", "baby,sports,syn1m").split(","):
        ds, _, _, _, _ = bench.build_problem(name, 2022, None)
        U, I, d = ds.n_users, ds.n_items, ds.embed_size
        g = torch.Generator(device=dev).manual_seed(7)
        ua = torch.randn(U, d, generator=g, device=dev)
        ia = torch.randn(I, d, generator=g, device=dev)
        excl = _device_csr(*train_rows(ds), dev)
        users = np.arange(U, dtype=np.int64)
        users_dev = torch.from_numpy(users).to(dev)
        for k in (int(x) for x in opt("--ks", "20,100").split(",")):
            rec = recommend.Recommender(ia, excl, k)
            ids = torch.empty(U, k, dtype=torch.int32, device=dev)
            sc = torch.empty(U, k, dtype=torch.float32, device=dev)
            ws = rec._key_ws(U)
            ms = timed(lambda: rec._launch(ua, users_dev, U, ids, sc, k, ws))
            del ws
            with tempfile.TemporaryDirectory() as tmp:
                rec.export(ua, users, tmp)                 # warm-up: page cache, pinned buffers
                t0 = time.perf_counter()
                rec.export(ua, users, tmp)
                export_s = time.perf_counter() - t0
            flop = 2.0 * U * I * d
            res["rows"].append(dict(config=name, users=U, items=I, d=d, k=k, route="shared-memory buffers" if k <= 64 else "wide buffers",
                                    rank_ms=round(ms, 3), users_per_s=round(U / ms * 1e3), export_s=round(export_s, 3),
                                    export_users_per_s=round(U / export_s), tflops=round(flop / (ms * 1e-3) / 1e12, 2),
                                    fraction_of_fp32_bound=round(flop / (ms * 1e-3) / FP32_BOUND, 3)))
            del rec, ids, sc
        del ua, ia, excl, users_dev
        torch.cuda.empty_cache()
    return res


def sharded():
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    pos = [a for a in sys.argv[1:] if not a.startswith("--") and a not in (opt("--k", None), opt("--iters", None), opt("--warmup", None))]
    name, k = (pos[0] if pos else "sports"), int(opt("--k", 20))
    ds, P_cpu, feats_cpu, _, _ = bench.build_problem(name, 2022, None)
    U, I, d = ds.n_users, ds.n_items, ds.embed_size
    cfg = HotStepConfig(embed_size=d, n_layers=ds.n_layers, batch_size=bench.BATCH)
    Pl, fl, gl, pu, pi = shard_problem(P_cpu, feats_cpu, ds.ui_norm, ds.iu_norm, rank, world, dev)
    step = RowShardedHotStep(Pl, fl, gl, cfg, bench.BATCH, pu, pi, rank)
    ip, ix = train_rows(ds)
    lo, hi = pu.bounds(rank)
    blk = np.full(pu.block + 1, ip[hi] - ip[lo], np.int64)
    blk[:hi - lo + 1] = ip[lo:hi + 1] - ip[lo]
    sr = recommend.ShardedRecommender((blk, ix[ip[lo]:ip[hi]]), pu, pi, rank, I, k, device=dev)
    users = np.arange(U, dtype=np.int64)
    mine = users[sr.mine(users)] - lo
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    tot = np.zeros(4)
    with tempfile.TemporaryDirectory() as tmp:
        for it in range(warmup + iters):
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            ev[0].record()
            u_f, i_f = step.final_embeddings()
            ev[1].record()
            items = sr.gather_items(i_f)
            ev[2].record()
            rec = sr.local(items)
            rec.topk(u_f, mine)
            ev[3].record()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rec._export(rec._user_table(u_f), mine, mine + lo, tmp, 1 << 16, recommend._rank_prefix(rank, world), it, [])
            export_ms = (time.perf_counter() - t0) * 1e3
            if it >= warmup:
                tot += [ev[j].elapsed_time(ev[j + 1]) for j in range(3)] + [export_ms]
            del u_f, i_f, items, rec
    ms = torch.tensor(tot / iters, device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    flop = 2.0 * (U / world) * I * d
    res = dict(mode="row-sharded", config=name, n_gpus=world, users=U, items=I, d=d, k=k, iters=iters,
               **dict(zip(("forward_ms", "item_allgather_ms", "rank_ms", "export_ms"), (round(float(v), 3) for v in ms))))
    res.update(users_per_s=round(U / float(ms[:3].sum() + ms[3]) * 1e3),
               rank_tflops_per_gpu=round(flop / (float(ms[2]) * 1e-3) / 1e12, 2))
    if world > 1:
        dist.destroy_process_group()
    return res


res = sharded() if "--sharded" in sys.argv else one_gpu()
res.update(card(), fp32_bound_tflops=FP32_BOUND / 1e12)
if rank == 0:
    print(json.dumps(res))
