"""Audience speed (audience.py): the top-k users of listed items against every user of a synthetic problem, seeded random fp32
tables, exclusion = the transposed training rows of the problem's graph.

    python tools/audience_bench.py [--configs baby,sports,syn1m] [--ks 20,100] [--counts 1,8,64,1024,all] [--iters K] [--warmup W]

Per config, k and count of listed items (the first items of a seeded permutation; "all" = every item):
  slices            the slice count Recommender._slices picks (1 = the unsliced sweep)
  rank_ms           the ranking as the library runs it: the sliced sweep and the merge when slices > 1 (CUDA events)
  unsliced_ms       the same call forced to the unsliced sweep (skipped when slices == 1: it is rank_ms)
  merge_ms          the merge of the partial lists alone (slices > 1)
  export_ms         the whole chunked export to a temporary directory (host clock after a synchronise)
  tflops / of_bound 2 * items * users * d FLOP over rank_ms, and that rate over the 67 TFLOP/s fp32 bound of the H100 SXM (the
                    sweep is fp32 FMA; a CTA scores 8 queries, so with fewer than 8 items it does 8 queries' work)
and the row-sharded path at world 1 (ShardedAudience on one rank, no process group): item gather, the rank's sweep, exchange and
merge, each timed alone.  One JSON line per workload, then one with the card name and power limit read in the same run.
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

from mmssl_b200 import audience, recommend  # noqa: E402
from mmssl_b200.evaluate import _device_csr  # noqa: E402
from mmssl_b200.parallel import RowPartition  # noqa: E402
from mmssl_b200.synthetic import CONFIGS, make_bipartite  # noqa: E402

FP32_BOUND = 67e12
opt = lambda k, dflt: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else dflt
iters, warmup = int(opt("--iters", 5)), int(opt("--warmup", 2))
configs = opt("--configs", "baby,sports,syn1m").split(",")
ks = [int(x) for x in opt("--ks", "20,100").split(",")]
counts = opt("--counts", "1,8,64,1024,all").split(",")
dev = torch.device("cuda")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(card=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip() if q.returncode == 0 else None)


def timed(fn, n_iter=None):
    """Mean ms of fn over the timed calls after the warm-up ones, CUDA events."""
    n_iter = n_iter or iters
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n_iter):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n_iter


def problem(name):
    U, I, nnz, d, *_ = CONFIGS[name]
    tr = make_bipartite(U, I, nnz, seed=3).tocsr()
    tr.sort_indices()
    rng = np.random.default_rng(2)
    ua = torch.from_numpy(rng.standard_normal((U, d), dtype=np.float32)).to(dev)
    ia = torch.from_numpy(rng.standard_normal((I, d), dtype=np.float32)).to(dev)
    return U, I, d, ua, ia, (tr.indptr.astype(np.int64), tr.indices.astype(np.int64)), rng.permutation(I).astype(np.int64)


def one_gpu(name, U, I, d, ua, ia, excl, perm, k):
    aud = audience.Audience(ua, excl, k)
    rec = aud.rec
    for c in counts:
        n = I if c == "all" else min(int(c), I)
        items = perm[:n]
        items_dev = torch.from_numpy(items).to(dev)
        ids = torch.empty(n, k, dtype=torch.int32, device=dev)
        sc = torch.empty(n, k, dtype=torch.float32, device=dev)
        ws = rec._key_ws(n)
        s = rec._slices(n)
        big = n * U * d > 2e12                  # a call of seconds: one timed call is enough
        row = dict(config=name, users=U, items=I, d=d, k=k, listed=n, slices=s)
        row["rank_ms"] = round(timed(lambda: rec._launch(ia, items_dev, n, ids, sc, k, ws), 1 if big else None), 3)
        if s > 1:
            chosen = (ids.clone(), sc.clone())
            rec._slices = lambda m: 1
            ws1 = rec._key_ws(n)
            row["unsliced_ms"] = round(timed(lambda: rec._launch(ia, items_dev, n, ids, sc, k, ws1)), 3)
            del rec._slices
            row["same_lists"] = bool(torch.equal(chosen[0], ids) and torch.equal(chosen[1].view(torch.int32), sc.view(torch.int32)))
            pid = torch.empty(s, n, k, dtype=torch.int32, device=dev)
            psc = torch.empty(s, n, k, dtype=torch.float32, device=dev)
            lib = recommend._lib.load()
            recommend._lib.check(lib.mmssl_recommend_topk_sliced(
                recommend.ptr(ia), d, recommend.ptr(ua), d, U, d, recommend.ptr(items_dev), n, recommend.ptr(excl[0]),
                recommend.ptr(excl[1]), k, s, recommend.ptr(pid), recommend.ptr(psc), recommend.ptr(ws), recommend.stream()))
            row["merge_ms"] = round(timed(lambda: recommend.merge_lists(pid, psc, n, s, k, k, n * k, ids, sc, k)), 4)
        with tempfile.TemporaryDirectory() as tmp:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            aud.export(ia, items, tmp)
            row["export_ms"] = round(1e3 * (time.perf_counter() - t0), 2)
        flops = 2.0 * n * U * d
        row["tflops"] = round(flops / (row["rank_ms"] * 1e-3) / 1e12, 3)
        row["of_bound"] = round(flops / (row["rank_ms"] * 1e-3) / FP32_BOUND, 4)
        print(json.dumps(row), flush=True)


def sharded_world1(name, U, I, d, ua, ia, excl_host, perm, k):
    """ShardedAudience at world 1: each step of _chunk timed alone (gather, the rank's sweep, exchange, merge)."""
    pu, pi = RowPartition(U, 1), RowPartition(I, 1)
    sa = audience.ShardedAudience(excl_host, pu, pi, 0, k, device=dev)
    rec = sa.local(ua)
    for c in ("1", "64"):
        n = int(c)
        items = np.sort(perm[:n])
        items_dev = torch.from_numpy(items).to(dev)
        part = torch.empty(n, 2 * k, dtype=torch.int32, device=dev)
        out_ids = torch.empty(n, k, dtype=torch.int32, device=dev)
        out_sc = torch.empty(n, k, dtype=torch.float32, device=dev)
        row = dict(config=name, path="sharded_world1", k=k, listed=n, slices=rec._slices(n))
        row["gather_ms"] = round(timed(lambda: sa.gather_items(ia)), 4)
        row["sweep_ms"] = round(timed(lambda: rec._launch(ia, items_dev, n, part, part[:, k:].view(torch.float32), 2 * k)), 3)
        row["exchange_ms"] = round(timed(lambda: sa.exchange(part, [n], [n])), 4)
        row["merge_ms"] = round(timed(lambda: recommend.merge_lists(part, part[:, k:].view(torch.float32), n, 1, k, 2 * k, n * 2 * k,
                                                                  out_ids, out_sc, k)), 4)
        got = sa.topk(ua, ia, items)
        want = audience.Audience(ua, sa.exclude, k).topk(ia, items)
        row["same_lists"] = bool(torch.equal(got[0], want[0]) and torch.equal(got[1].view(torch.int32), want[1].view(torch.int32)))
        print(json.dumps(row), flush=True)


def main():
    for name in configs:
        U, I, d, ua, ia, train, perm = problem(name)
        excl_host = audience.transpose_csr(*train, I)
        excl = _device_csr(*excl_host, dev)
        for k in ks:
            one_gpu(name, U, I, d, ua, ia, excl, perm, k)
            sharded_world1(name, U, I, d, ua, ia, excl_host, perm, k)
        del ua, ia, excl
        torch.cuda.empty_cache()
    print(json.dumps(dict(card(), sms=torch.cuda.get_device_properties(0).multi_processor_count)), flush=True)


if __name__ == "__main__":
    main()
