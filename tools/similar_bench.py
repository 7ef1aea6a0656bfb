"""Similar-items throughput (similar.py: mmssl_unit_rows + mmssl_recommend_topk): items ranked per second over every item of a
catalogue of the shape of baby / sports / syn1m (synthetic.CONFIGS: items and embedding width), "model" space, on a seeded random
fp32 table.

    python tools/similar_bench.py [--configs baby,sports,syn1m] [--ks 20,100] [--iters K] [--warmup W]
        per config: the unit-row kernel alone; per config and k: the ranking kernel alone over every item (CUDA events), and
        the whole chunked export to a temporary directory (unit rows, ranking, device-to-host copies and file writes)

Reports the algorithmic work of the ranking, 2 * items * items * d FLOP, over its kernel time against the 67 TFLOP/s fp32
CUDA-core bound of the H100 SXM (the sweep is fp32 FMA), and the unit-row kernel's bytes (read + write of the table) over its
time.  One JSON line in the shape of tools/recommend_bench.py's, with the card name and power limit read in the same run.  Not
part of bench.py's contract; H100 numbers in DESIGN section 6."""
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

from mmssl_b200 import ops, similar  # noqa: E402
from mmssl_b200.synthetic import CONFIGS  # noqa: E402

FP32_BOUND = 67e12
opt = lambda k, dflt: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else dflt
iters, warmup = int(opt("--iters", 3)), int(opt("--warmup", 1))
dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return dict(card=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip() if q.returncode == 0 else None)


def timed(fn, n=None):
    """Mean ms of fn over `n` (default `iters`) calls after `warmup`, CUDA events."""
    n = n or iters
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    res = {"mode": "one GPU", "space": "model", "iters": iters, "rows": [], "unit_rows": []}
    for name in opt("--configs", "baby,sports,syn1m").split(","):
        _, I, _, d, *_ = CONFIGS[name]
        g = torch.Generator(device=dev).manual_seed(7)
        table = torch.randn(I, d, generator=g, device=dev)
        unit = torch.empty_like(table)
        ms_unit = timed(lambda: ops.unit_rows(table, unit), n=max(iters, 100))
        res["unit_rows"].append(dict(config=name, items=I, d=d, ms=round(ms_unit, 4),
                                     gb_per_s=round(2 * I * d * 4 / (ms_unit * 1e-3) / 1e9, 1)))
        items = np.arange(I, dtype=np.int64)
        items_dev = torch.from_numpy(items).to(dev)
        for k in (int(x) for x in opt("--ks", "20,100").split(",")):
            sim = similar.SimilarItems(table, k)
            rec = sim.rec
            ids = torch.empty(I, k, dtype=torch.int32, device=dev)
            sc = torch.empty(I, k, dtype=torch.float32, device=dev)
            ws = rec._key_ws(I)
            ms = timed(lambda: rec._launch(sim.unit, items_dev, I, ids, sc, k, ws))
            del ws
            with tempfile.TemporaryDirectory() as tmp:
                similar.SimilarItems(table, k).export(items, tmp)        # warm-up: page cache, pinned buffers
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                similar.SimilarItems(table, k).export(items, tmp)
                export_s = time.perf_counter() - t0
            flop = 2.0 * I * I * d
            res["rows"].append(dict(config=name, items=I, d=d, k=k, route="shared-memory buffers" if k <= 64 else "wide buffers",
                                    rank_ms=round(ms, 3), items_per_s=round(I / ms * 1e3), export_s=round(export_s, 3),
                                    export_items_per_s=round(I / export_s), tflops=round(flop / (ms * 1e-3) / 1e12, 2),
                                    fraction_of_fp32_bound=round(flop / (ms * 1e-3) / FP32_BOUND, 3)))
            del sim, rec, ids, sc
        del table, unit, items_dev
        torch.cuda.empty_cache()
    return res


if __name__ == "__main__":
    torch.cuda.set_device(dev)
    out = main()
    out.update(card(), fp32_bound_tflops=FP32_BOUND / 1e12)
    print(json.dumps(out))
