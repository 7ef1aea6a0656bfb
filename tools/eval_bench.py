"""Evaluation of every user of a synthetic dataset (synthetic.make_bipartite training rows, 1..8 held-out items per user
drawn from a seed, random fp32 embeddings) in part mode (top-K ranking + metrics) and full mode (the same plus the
per-user ROC-AUC over all non-training items), timed with CUDA events after a warm-up.  Prints one JSON line with the
card name and power limit read in the same run.

    python tools/eval_bench.py [baby|sports|tiktok] [--iters N] [--warmup W] [--ks "[10, 20, 50, 100]"]

--ks takes the reference's --Ks syntax; up to 8 cut-offs of at most 64 use the shared-memory kernel, any other list the
wide path (mmssl_eval_rank_wide).

Not part of bench.py's contract; H100 numbers in DESIGN section 6."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("config", nargs="?", default="baby", choices=["tiktok", "baby", "sports"])
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--ks", default="[10, 20, 50]")
a = ap.parse_args()
Ks = [int(k) for k in json.loads(a.ks)]

from mmssl_b200.evaluate import Evaluator  # noqa: E402
from mmssl_b200.synthetic import CONFIGS, make_bipartite  # noqa: E402

U, I, nnz, d, *_ = CONFIGS[a.config]
tr = make_bipartite(U, I, nnz, seed=3).tocsr()
tr.sort_indices()
rng = np.random.default_rng(a.seed)
train = {u: tr.indices[tr.indptr[u]:tr.indptr[u + 1]].tolist() for u in range(U) if tr.indptr[u + 1] > tr.indptr[u]}
held = {u: rng.choice(I, size=int(rng.integers(1, 9)), replace=False).tolist() for u in range(U)}
dev = torch.device("cuda")
ua = torch.randn(U, d, generator=torch.Generator().manual_seed(a.seed)).to(dev)
ia = torch.randn(I, d, generator=torch.Generator().manual_seed(a.seed + 1)).to(dev)
users = list(range(U))


def time_mode(flag):
    ev = Evaluator(train, held, {}, U, I, Ks, test_flag=flag)
    for _ in range(a.warmup):
        ev.rank(ua, ia, users, False)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(a.iters):
        out = ev.rank(ua, ia, users, False)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / a.iters, out


part_ms, part = time_mode("part")
full_ms, full = time_mode("full")
same = all(torch.equal(part[k], full[k]) for k in ("ranked", "hits", "per_user"))
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print(json.dumps(dict(config=a.config, users=U, items=I, d=d, Ks=Ks, wide=bool(Evaluator(train, held, {}, U, I, Ks).wide), iters=a.iters, part_ms=round(part_ms, 3), full_ms=round(full_ms, 3),
                      full_over_part=round(full_ms / part_ms, 3), ranking_equal=same,
                      mean_auc=float(full["auc"].mean().item()), card=torch.cuda.get_device_name(),
                      nvidia_smi=q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None)))
