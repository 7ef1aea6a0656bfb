"""Large batches on one H100: device-sampler time, InfoNCE forward + backward time and hot-step time at batch sizes above the
reference's default of 1024.  Prints the card's name and power limit from the same run, then one JSON line per measurement.

  sampler : DeviceTripleSampler.sample_into at B in {1024, 4096, 16384} on Baby and syn1m (1M users).  B = 1024 takes the
            one-CTA kernel, larger batches the multi-CTA radix select over all n_exist users (O(n_exist) per call).
  infonce : ops.infonce_forward + ops.infonce_backward at n in {1024, ..., 16384}, d in {64, 128}: the CUDA-core kernels
            ("simt") at every n and the stored-exponential tensor-core kernels ("tc") where mmssl_infonce_tc_supported.  For
            "tc" the issued tensor-core work (three bf16 MMAs per product, n padded to 128: 42 n^2 d flop per forward +
            backward) over the median time is set against the 989 TFLOP/s dense-bf16 data-sheet rate.
  hotstep : captured hot step with the optimiser, ms/step at Baby and Sports with B in {1024, 4096, 16384}: host batches
            (copied in per step), the device sampler's batches drawn ahead and copied in the same way, and the device sampler
            inside the graph.  Before timing, one step of each from the same
            parameters on the same triples (the host trainer is fed the device sampler's first batch): loss terms and
            gradients must agree.
CUDA-event medians after a warm-up.

    python tools/large_batch_bench.py [--sections sampler,infonce,hotstep] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

BF16_PEAK = 989e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def event_times_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        ts.append((a, b))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ts]


def summary(ms):
    return {"median_ms": round(statistics.median(ms), 5), "min_ms": round(min(ms), 5), "max_ms": round(max(ms), 5), "reps": len(ms)}


def bench_sampler(emit, reps):
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import make_dataset
    for name in ("baby", "syn1m"):
        ds = make_dataset(name)
        smp = DeviceTripleSampler(ds.train, seed=1)
        step = torch.zeros(1, dtype=torch.int32, device="cuda")
        for B in (1024, 4096, 16384):
            out = torch.empty(3, B, dtype=torch.int64, device="cuda")

            def call():
                step.add_(1)
                smp.sample_into(out, step_dev=step)
            ms = event_times_ms(call, reps)
            emit({"section": "sampler", "config": name, "n_exist": smp.exist.numel(), "batch": B,
                  "path": "one-CTA" if B <= 1024 else "multi-CTA select", **summary(ms)})


def bench_infonce(emit, reps):
    from mmssl_b200 import ops
    for d in (64, 128):
        for n in (1024, 2048, 4096, 8192, 16384):
            torch.manual_seed(n + d)
            z1, z2 = torch.randn(n, d, device="cuda"), torch.randn(n, d, device="cuda")
            g1, g2 = torch.zeros(n, d, device="cuda"), torch.zeros(n, d, device="cuda")
            seed = torch.ones(1, device="cuda")
            for impl in ("tc", "simt"):
                w = ops.InfoNCEWork(n, d, "cuda", impl=impl)
                if impl == "tc" and not w.tc:
                    continue

                def call():
                    ops.infonce_forward(z1, z2, None, 2.0, w, g_loss=seed)
                    ops.infonce_backward(None, 2.0, w, g1, g2)
                ms = event_times_ms(call, reps if n <= 4096 else max(5, reps // 4))
                rec = {"section": "infonce", "impl": impl, "n": n, "d": d, **summary(ms)}
                if impl == "tc":
                    npad = (n + 127) // 128 * 128
                    rate = 42.0 * npad * npad * d / (statistics.median(ms) * 1e-3)
                    rec.update(issued_tflops=round(rate / 1e12, 2), share_of_bf16_datasheet=round(rate / BF16_PEAK, 4))
                emit(rec)
                del w


def bench_hotstep(emit, steps):
    import bench
    from mmssl_b200.engine import LIVE
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import TripleSampler
    dev = torch.device("cuda")
    for name in ("baby", "sports"):
        ds, P, feats, graphs, _ = bench.build_problem(name, 2022, dev)
        for B in (1024, 4096, 16384):
            cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=B)
            host = bench.HotStepTrainer({k: v.clone() for k, v in P.items()}, feats, graphs, cfg, B)
            devs = bench.HotStepTrainer({k: v.clone() for k, v in P.items()}, feats, graphs, cfg, B,
                                        sampler=DeviceTripleSampler(ds.train, device=dev, seed=7))
            # the capture's warm-up steps advanced both optimisers from the same parameters, but on different batches:
            # restart both from P before the comparison step
            for tr in (host, devs):
                for k in LIVE:
                    tr.hs.P[k].copy_(P[k]); tr.hs.m[k].zero_(); tr.hs.v[k].zero_()
                tr.hs.step_dev.zero_()
            torch.manual_seed(3)
            loss_d = devs.train_step_device_sampled()
            idx = devs.hs.idx.cpu()
            torch.manual_seed(3)
            loss_h = host.train_step(idx[0], idx[1], idx[2])
            diff_out5 = float((host.hs.out5 - devs.hs.out5).abs().max())
            diff_grad = max(float((host.hs.grads[k] - devs.hs.grads[k]).abs().max()) for k in LIVE)
            sampler_host = TripleSampler(ds.train, seed=3)
            batches = [sampler_host.sample(B) for _ in range(steps)]
            # the device sampler's batches, drawn ahead and copied in like host batches: separates what the batches are
            # from what drawing them inside the graph costs
            pre, buf = DeviceTripleSampler(ds.train, device=dev, seed=11), torch.empty(3, B, dtype=torch.int64, device=dev)
            dev_batches = []
            for i in range(steps):
                pre.sample_into(buf, step=i)
                dev_batches.append(tuple(t.cpu().numpy() for t in buf))
            for label, run in (("host_batches", lambda i: host.train_step(*batches[i % len(batches)])),
                               ("device_sampler_batches_copied_in", lambda i: host.train_step(*dev_batches[i % len(dev_batches)])),
                               ("device_sampler", lambda i: devs.train_step_device_sampled())):
                for i in range(3):
                    run(i)
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(steps):
                    run(i)
                b.record()
                torch.cuda.synchronize()
                emit({"section": "hotstep", "config": name, "batch": B, "input": label, "ms_per_step": round(a.elapsed_time(b) / steps, 4),
                      "steps": steps, "first_step_loss_host": loss_h, "first_step_loss_device": loss_d,
                      "max_abs_diff_loss_terms": diff_out5, "max_abs_diff_grads": diff_grad})
            del host, devs
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", default="sampler,infonce,hotstep")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("large_batch_bench needs the GPU")
    sink = open(a.out, "w") if a.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")
            sink.flush()
    emit({"card": card()})
    secs = a.sections.split(",")
    if "sampler" in secs:
        bench_sampler(emit, a.reps)
    if "infonce" in secs:
        bench_infonce(emit, a.reps)
    if "hotstep" in secs:
        bench_hotstep(emit, a.steps)


if __name__ == "__main__":
    main()
