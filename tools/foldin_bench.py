"""Fold-in speed (foldin.py): fold item lists into user rows and rank them, on seeded random fp32 tables of a synthetic problem.

    python tools/foldin_bench.py [--configs baby,sports,syn1m] [--counts 1,64,4096,65536] [--k 20] [--iters K] [--warmup W]

Queries are the training rows of random users of the problem's graph, with those users' ids (a trained user with fresh
interactions: u_0 is gathered too); the last workload per config is long rows of 10^4 random items without ids (where the config
has that many items).  K = the config's layer count.  Per workload:
  fold_ms        mmssl_fold_users alone (CUDA events, mean over the timed launches after the warm-up ones)
  fold_rank_ms   the fold and the ranking of the folded rows (Recommender's sweep, sliced for few queries) from device arrays
  fold_share     fold_ms / fold_rank_ms
  queries_per_s  queries / fold_rank_ms
  gathered_mb / effective_gbs   sum |r| (K + 2) d 4 + n d 4 (2 with an id, else 1) bytes, and that over fold_ms -- an effective
                 rate: the item tables of Baby and Sports fit the 50 MB L2, so it is not an HBM figure there
One JSON line per workload, then one with the card name and power limit read in the same run.  Not part of bench.py's contract;
H100 numbers in DESIGN section 6."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mmssl_b200 import _lib, foldin  # noqa: E402
from mmssl_b200.recommend import Recommender  # noqa: E402
from mmssl_b200.synthetic import CONFIGS, make_bipartite  # noqa: E402

opt = lambda k, dflt: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else dflt
iters, warmup = int(opt("--iters", 20)), int(opt("--warmup", 3))
configs = opt("--configs", "baby,sports,syn1m").split(",")
counts = [int(c) for c in opt("--counts", "1,64,4096,65536").split(",")]
K_TOP = int(opt("--k", 20))
LONG = 10_000
dev = torch.device("cuda")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(card=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip() if q.returncode == 0 else None)


def timed(fn):
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


def workload(name, fi, q, users, K):
    n = users.size
    ip, ix = torch.from_numpy(q[0]).to(dev), torch.from_numpy(q[1]).to(dev)
    w = torch.from_numpy(foldin.row_weights(np.diff(q[0]))).to(dev)
    us = torch.from_numpy(users).to(dev)
    out = torch.empty(n, fi.d, dtype=torch.float32, device=dev)
    lib = _lib.load()
    fold = lambda: _lib.check(lib.mmssl_fold_users(_lib.ptr(ip), _lib.ptr(ix), _lib.ptr(us), _lib.ptr(w), n, _lib.ptr(fi.u0),
                                                   fi.u0.stride(0), fi._desc, fi.d, K, 1.0 / (K + 1), fi.rate, _lib.ptr(out),
                                                   out.stride(0), _lib.stream()))
    rec = Recommender(fi.items, (ip, ix), K_TOP)
    ids = torch.empty(n, K_TOP, dtype=torch.int32, device=dev)
    sc = torch.empty(n, K_TOP, dtype=torch.float32, device=dev)
    rows = torch.arange(n, dtype=torch.int64, device=dev)
    ws = rec._key_ws(n)

    def both():
        fold()
        rec._launch(out, rows, n, ids, sc, K_TOP, ws)

    f_ms, fr_ms = timed(fold), timed(both)
    nnz = int(q[0][-1])
    gathered = nnz * (K + 2) * fi.d * 4 + n * fi.d * 4 * (2 if (users >= 0).any() else 1)
    got = fi.topk(q, K_TOP, users, "train")
    row = dict(config=name, items=fi.n_items, d=fi.d, K=K, queries=n, mean_row=round(nnz / max(n, 1), 1), slices=rec._slices(n),
               fold_ms=round(f_ms, 4), fold_rank_ms=round(fr_ms, 4), fold_share=round(f_ms / fr_ms, 4),
               queries_per_s=round(n / (fr_ms * 1e-3)), gathered_mb=round(gathered / 1e6, 2),
               effective_gbs=round(gathered / (f_ms * 1e-3) / 1e9, 1), lists_ok=bool((got[0] >= -1).all()))
    print(json.dumps(row), flush=True)


def main():
    for name in configs:
        U, I, nnz, d, K, *_ = CONFIGS[name]
        g = make_bipartite(U, I, nnz, seed=3).tocsr()
        g.sort_indices()
        rng = np.random.default_rng(2)
        t = lambda n: torch.from_numpy(rng.standard_normal((n, d), dtype=np.float32)).to(dev)
        fi = foldin.FoldIn(t(U), [t(I) for _ in range(K)], t(I), t(I), t(I))
        train = (g.indptr.astype(np.int64), g.indices.astype(np.int64))
        for n in counts:
            users = rng.integers(0, U, n).astype(np.int64)
            workload(name, fi, foldin.take_rows(train, users), users, K)
        if I >= LONG:
            for n in (1, 64, 4096):
                ix = np.concatenate([np.sort(rng.choice(I, LONG, replace=False)) for _ in range(n)]).astype(np.int64)
                workload(name + "_long", fi, (np.arange(n + 1, dtype=np.int64) * LONG, ix), np.full(n, -1, np.int64), K)
        del fi
        torch.cuda.empty_cache()
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
