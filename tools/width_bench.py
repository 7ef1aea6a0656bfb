"""Time per embedding width: the captured hot step (forward, backward, fused losses, AdamW; B = 1024), the SpMM A_ui X and the
grouped projection forward (image and text in one launch), at the Baby and Sports shapes, for d in {32, 64, 96, 128, 192, 256}.
CUDA events, medians after a warm-up; the card name and power limit are read in the same run.

    python tools/width_bench.py [--configs baby,sports] [--widths 32,64,96,128,192,256] [--steps 30] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tools.proj_bench import card  # noqa: E402


def median_ms(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def problem_at_width(name, d, dev):
    """bench.build_problem with the dataset's embedding width replaced by d (same graphs and features)."""
    import bench
    from mmssl_b200 import synthetic
    real = synthetic.make_dataset

    def at_width(*a, **k):
        ds = real(*a, **k)
        ds.embed_size = d
        return ds
    synthetic.make_dataset = at_width
    try:
        return bench.build_problem(name, 2022, dev)
    finally:
        synthetic.make_dataset = real


def measure(name, d, steps, batch, dev):
    from mmssl_b200 import ops
    from mmssl_b200.engine import P_WT, P_WV
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.synthetic import TripleSampler
    ds, P, feats, graphs, _ = problem_at_width(name, d, dev)
    cfg = HotStepConfig(embed_size=d, n_layers=ds.n_layers, batch_size=batch)
    hs = HotStep(P, feats, list(graphs), cfg, batch=batch)
    hs.set_indices(*TripleSampler(ds.train, seed=3).sample(batch))
    hs.capture(warmup=2)
    step = median_ms(hs.replay, steps)
    x = torch.randn(ds.n_items, d, device=dev)
    y = torch.empty(ds.n_users, d, device=dev)
    spmm = median_ms(lambda: ops.spmm(graphs[0].fwd, [x], [y]), 5 * steps)
    max_ctas = hs.engine.proj_max_ctas
    splits, floats = ops.gemm_bf16x3_group_plan([(fs.n_items, d, fs.dim) for fs in feats], max_ctas)
    parts = torch.empty(sum(floats), device=dev).split(floats)
    probs = []
    for w, fs, sk, part in zip((P[P_WV], P[P_WT]), feats, splits, parts):
        w_hi, w_lo = ops.split_bf16(w)
        probs.append((fs.hi, fs.lo, w_hi, w_lo, fs.n_items, d, fs.dim, sk, part))
    proj = median_ms(lambda: ops.gemm_bf16x3_group(probs, max_ctas), 5 * steps)
    return dict(config=name, d=d, batch=batch, hot_step_ms=round(step, 4), spmm_ui_x_ms=round(spmm, 4), proj_fwd_group_ms=round(proj, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="baby,sports")
    ap.add_argument("--widths", default="32,64,96,128,192,256")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda")
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for name in a.configs.split(","):
        for d in (int(w) for w in a.widths.split(",")):
            r = measure(name, d, a.steps, a.batch, dev)
            rows.append(r)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
