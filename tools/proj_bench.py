"""Projection GEMM timing per direction (forward X = F W^T, weight gradient dW^T = F^T dX), image and text together, in
three forms:
  streams : the two single-problem launches (mmssl_gemm_bf16x3) on two streams, forked and joined as engine.py did;
  grouped : one grouped persistent launch (mmssl_gemm_bf16x3_group), when the library has it;
  alone   : each GEMM by itself, for the record.
CUDA events over many launches after a warm-up; before every launch the L2 is flushed by READING a 192 MiB buffer (a
write-flush would leave dirty lines whose write-back lands inside the timed window).  Rates are algorithmic bytes,
4 M K + 4 N K + 4 M N per problem (bf16 hi + lo operands, fp32 partials), over the median time.

    python tools/proj_bench.py [--configs baby,sports,syn1m] [--reps 40] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers stay meaningful with the torch name alone
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def timed(fn, flush, sink, reps, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        torch.sum(flush, dim=0, out=sink)   # read-only L2 flush
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        ts.append((a, b))
    torch.cuda.synchronize()
    us = [a.elapsed_time(b) * 1e3 for a, b in ts]
    return statistics.median(us), min(us), max(us)


def problems(name, dev):
    from mmssl_b200 import ops
    from mmssl_b200.synthetic import CONFIGS
    _, I, _, d, _, dv, dt = CONFIGS[name]
    g = torch.Generator(device=dev).manual_seed(1)
    fwd, wgrad = [], []
    for D in (dv, dt):
        f = torch.rand(I, D, device=dev, generator=g)
        f_hi, f_lo = ops.split_bf16(f)
        t_hi, t_lo = ops.split_bf16_t(f)
        del f
        w_hi, w_lo = ops.split_bf16(torch.randn(d, D, device=dev, generator=g) * 0.02)
        gx_hi, gx_lo = ops.split_bf16_t(torch.randn(I, d, device=dev, generator=g) * 1e-3, ldo=t_hi.shape[1])
        fwd.append([f_hi, f_lo, w_hi, w_lo, I, d, D])
        wgrad.append([t_hi, t_lo, gx_hi, gx_lo, D, d, I])
    return fwd, wgrad


def bench_direction(probs, flush, sink, reps, dev, max_ctas=(0,)):
    from mmssl_b200 import ops
    alg = sum(4 * m * k + 4 * n * k + 4 * m * n for (_, _, _, _, m, n, k) in probs)
    out = {"shapes": [[m, n, k] for (_, _, _, _, m, n, k) in probs], "algorithmic_bytes": alg}
    single = []
    for (a_hi, a_lo, b_hi, b_lo, m, n, k) in probs:
        floats, sk = ops.gemm_bf16x3_plan(m, n, k)
        single.append((a_hi, a_lo, b_hi, b_lo, m, n, k, sk, torch.empty(floats, device=dev)))
    side = torch.cuda.Stream(device=dev)

    def streams():
        cur = torch.cuda.current_stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            ops.gemm_bf16x3(*single[1])
        ops.gemm_bf16x3(*single[0])
        cur.wait_stream(side)

    def rec(key, fn, nbytes):
        med, lo, hi = timed(fn, flush, sink, reps)
        out[key] = {"us": round(med, 2), "us_min": round(lo, 2), "us_max": round(hi, 2), "tb_s": round(nbytes / (med * 1e-6) / 1e12, 3)}

    rec("streams", streams, alg)
    out["streams"]["splits"] = [q[7] for q in single]
    for cap in (max_ctas if hasattr(ops, "gemm_bf16x3_group") else []):
        splits, floats = ops.gemm_bf16x3_group_plan([(m, n, k) for (_, _, _, _, m, n, k) in probs], cap)
        parts = torch.empty(sum(floats), device=dev).split(floats)
        grouped = [tuple(p) + (sk, part) for p, sk, part in zip(probs, splits, parts)]
        key = "grouped" if cap == 0 else f"grouped_cap{cap}"
        rec(key, lambda: ops.gemm_bf16x3_group(grouped, cap), alg)
        out[key]["splits"] = splits
    for i, q in enumerate(single):
        m, n, k = q[4], q[5], q[6]
        rec(f"alone_{i}", lambda q=q: ops.gemm_bf16x3(*q), 4 * m * k + 4 * n * k + 4 * m * n)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="baby,sports,syn1m")
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--out", default=None)
    ap.add_argument("--max-ctas", default="0", help="grid caps of the grouped launch to time, comma-separated (0 = one resident wave)")
    a = ap.parse_args()
    from mmssl_b200 import _lib
    _lib.load(require_device=True)
    dev = torch.device("cuda")
    flush = torch.ones(192 * 1024 * 1024 // 4, device=dev)
    sink = torch.empty((), device=dev)
    res = {"card": card(), "flush": "read of 192 MiB before every launch", "configs": {}}
    print("card:", res["card"])
    for name in a.configs.split(","):
        fwd, wgrad = problems(name, dev)
        caps = [int(c) for c in a.max_ctas.split(",")]
        res["configs"][name] = {"fwd": bench_direction(fwd, flush, sink, a.reps, dev, caps),
                                "wgrad": bench_direction(wgrad, flush, sink, a.reps, dev, caps)}
        for direction, r in res["configs"][name].items():
            forms = [k for k in r if k == "streams" or k.startswith("grouped") or k.startswith("alone")]
            print(f"{name:7s} {direction:5s} " + "  ".join(f"{k} {r[k]['us']:8.1f} us {r[k]['tb_s']:5.2f} TB/s" for k in forms))
        del fwd, wgrad
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
