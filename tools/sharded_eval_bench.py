"""Evaluation of a row-sharded model on the N GPUs that hold it (evaluate.ShardedEvaluator, RowShardedHotStep.final_embeddings):
every user of a synthetic problem (bench.build_problem: tiktok / baby / sports / syn1m; training rows = its graph, 1..8 held-out
items per user drawn from a seed), part and full mode.  Phases timed with CUDA events after a warm-up, max over ranks:
the eval-mode forward, the item all-gather, the ranking of the rank's users, the gather of the per-user rows + the reduction.
With `check`, rank 0 also runs the one-GPU Evaluator on the all-gathered tables and reports whether the result, the AUC and
every ranked list (gathered from all ranks) are bitwise equal.  One JSON line from rank 0, with the card name and power limit
read in the same run.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/sharded_eval_bench.py [config] [check] [mc]
        [--iters K] [--warmup W] [--ks "[10, 20, 50]"]          (mc: the step's exchange through the multicast publish kernel)

Not part of bench.py's contract; H100 numbers in DESIGN section 5."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402
from mmssl_b200.evaluate import Evaluator, ShardedEvaluator  # noqa: E402
from mmssl_b200.hotstep import HotStepConfig  # noqa: E402
from mmssl_b200.parallel import all_gather_rows  # noqa: E402
from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
opt = lambda k, dflt: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else dflt
args = [a for a in args if a not in (opt("--iters", None), opt("--warmup", None), opt("--ks", None))]
name = args[0] if args and args[0] not in ("check", "mc") else "tiktok"
if name not in ("tiktok", "baby", "sports", "syn1m"):
    raise SystemExit(f"config must be tiktok, baby, sports or syn1m, not {name!r}")
check = "check" in args
iters, warmup = int(opt("--iters", 3)), int(opt("--warmup", 1))
Ks = [int(k) for k in json.loads(opt("--ks", "[10, 20, 50]"))]
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)

ds, P_cpu, feats_cpu, _, _ = bench.build_problem(name, 2022, None)           # the same seeded problem on every rank (host)
U, I = ds.n_users, ds.n_items
cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=bench.BATCH)
Pl, fl, gl, pu, pi = shard_problem(P_cpu, feats_cpu, ds.ui_norm, ds.iu_norm, rank, world, dev)
mode = "multicast" if "mc" in args and world > 1 else "nccl"
step = RowShardedHotStep(Pl, fl, gl, cfg, bench.BATCH, pu, pi, rank, exchange=mode)

# held-out rows: 1..8 distinct items per user from a seed (drawn with replacement, repeats within a row dropped)
rng = np.random.default_rng(0)
lens = rng.integers(1, 9, U)
row = np.repeat(np.arange(U, dtype=np.int64), lens)
key = np.unique(row * I + rng.integers(0, I, row.size))
h_row, h_idx = key // I, key % I
h_ptr = np.concatenate([[0], np.cumsum(np.bincount(h_row, minlength=U))]).astype(np.int64)
tr = ds.train.tocsr()
tr.sort_indices()


def block(indptr, indices):
    """The rank's user block of a CSR (indptr rebased, padding rows empty)."""
    lo, hi = pu.bounds(rank)
    ip = np.full(pu.block + 1, indptr[hi] - indptr[lo], np.int64)
    ip[:hi - lo + 1] = indptr[lo:hi + 1] - indptr[lo]
    return ip, indices[indptr[lo]:indptr[hi]]


train_blk, held_blk = block(tr.indptr.astype(np.int64), tr.indices), block(h_ptr, h_idx)
users = list(range(U))
res = {"config": name, "n_gpus": world, "users": U, "items": I, "d": ds.embed_size, "Ks": Ks, "users_evaluated": U,
       "exchange": "publish kernel over NVSwitch multicast / peer stores (no NCCL)" if mode == "multicast" else "NCCL",
       "schedule": step.schedule, "iters": iters}
ev1 = None
for flag in ("part", "full"):
    se = ShardedEvaluator(train_blk, held_blk, held_blk, pu, pi, rank, I, Ks, flag, device=dev)
    ids = se.check_users(users)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    tot = np.zeros(4)
    for it in range(warmup + iters):
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        ev[0].record()
        u_f, i_f = step.final_embeddings()
        ev[1].record()
        items = se.gather_items(i_f)
        ev[2].record()
        loc, mine = se.rank_local(u_f, items, ids, False)
        ev[3].record()
        out = se.combine(loc, ids)
        ev[4].record()
        torch.cuda.synchronize()
        if it >= warmup:
            tot += [ev[j].elapsed_time(ev[j + 1]) for j in range(4)]
    ms = torch.tensor(tot / iters, device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    phases = dict(zip(("forward_ms", "item_allgather_ms", "rank_ms", "rows_gather_reduce_ms"), (round(float(v), 3) for v in ms)))
    res[flag] = dict(phases, total_ms=round(float(ms.sum()), 3))
    if flag == "full":
        res["full"]["mean_auc"] = float(out["auc"].mean())
    if check:
        # every rank's ranked lists, padded to the largest count, gathered by position
        kmax = max(Ks)
        m = max(int(np.bincount(ids // pu.block, minlength=world).max()), 1)
        mine_rows = torch.full((m, 3 * kmax + 1), -1, dtype=torch.int32, device=dev)
        k = len(mine)
        mine_rows[:k, :kmax] = loc["ranked"]
        mine_rows[:k, kmax:2 * kmax] = loc["ranked_scores"].view(torch.int32)
        mine_rows[:k, 2 * kmax:3 * kmax] = loc["hits"]
        mine_rows[:k, 3 * kmax] = torch.from_numpy(mine.astype(np.int32)).to(dev)
        every = torch.empty(world * m, 3 * kmax + 1, dtype=torch.int32, device=dev) if world > 1 else mine_rows
        u_full = all_gather_rows(u_f, pu, None)
        if world > 1:
            dist.all_gather_into_tensor(every, mine_rows)
        if rank == 0:
            every = every[every[:, 3 * kmax] >= 0]
            pos = every[:, 3 * kmax].long()
            t = lambda ip, ix: (torch.from_numpy(ip).to(dev), torch.from_numpy(np.asarray(ix, np.int64)).to(dev))
            h = t(h_ptr, h_idx)
            one = Evaluator._from_csr(t(tr.indptr.astype(np.int64), tr.indices), h, h, U, I, Ks, dev, flag)
            want = one.rank(u_full, items, users, False)
            bits = lambda x: x.contiguous().view(torch.uint8)
            same = dict(result=torch.equal(bits(want["result"]), bits(out["result"])),
                        per_user=torch.equal(bits(want["per_user"]), bits(out["per_user"])),
                        ranked_lists=int(pos.numel()) == U and torch.equal(want["ranked"][pos], every[:, :kmax])
                        and torch.equal(want["ranked_scores"][pos].view(torch.int32), every[:, kmax:2 * kmax])
                        and torch.equal(want["hits"][pos], every[:, 2 * kmax:3 * kmax]))
            if flag == "full":
                same["auc"] = torch.equal(bits(want["auc"]), bits(out["auc"]))
            res[flag]["bitwise_equal_to_1gpu_evaluator"] = same
            del one, want
        del u_full, every
    del se, out, loc, items, u_f, i_f
if check and rank == 0:
    res["check"] = all(all(res[f]["bitwise_equal_to_1gpu_evaluator"].values()) for f in ("part", "full"))
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
res.update(card=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None)
if rank == 0:
    print(json.dumps(res))
if world > 1:
    dist.destroy_process_group()
