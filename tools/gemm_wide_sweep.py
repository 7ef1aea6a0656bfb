"""Error and time of the wide wgmma GEMM (csrc/gemm_wide.cu) against the accumulation-pass length, next to fp32 cuBLAS.
    python tools/gemm_wide_sweep.py          (on the GPU; prints one JSON line per shape)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from mmssl_b200 import ops  # noqa: E402


def timed(fn, reps=5):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def errs(got, want):
    diff = (got.double() - want).abs()
    mx = float(want.abs().max())
    return float(diff.max()) / mx, float((diff / (1e-4 * want.abs() + 1e-6 * mx)).max())


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    for (m, n, k) in [(2048, 1762, 7050), (1762, 7050, 2048), (2048, 7050, 1762)]:
        g = torch.Generator().manual_seed(m + n + k)
        a, b = torch.randn(m, k, generator=g).cuda(), torch.randn(n, k, generator=g).cuda()
        want = a.double() @ b.double().t()
        a_hi, a_lo = ops.split_bf16(a)
        b_hi, b_lo = ops.split_bf16(b)
        out = torch.empty(m, n, device="cuda")
        res = {"shape": [m, n, k], "gflop": round(2 * m * n * k / 1e9, 1)}
        ref = a @ b.t()
        e = errs(ref, want)
        res["cublas_fp32"] = {"max_norm_err": e[0], "elem_err": e[1], "ms": round(timed(lambda: torch.matmul(a, b.t(), out=out)), 4)}
        out2 = torch.empty(m, n, device="cuda")
        ops.sgemm(a, b, out2, trans_b=True)
        e = errs(out2, want)
        res["sgemm_simt"] = {"max_norm_err": e[0], "elem_err": e[1], "ms": round(timed(lambda: ops.sgemm(a, b, out2, trans_b=True)), 4)}
        for chunk in (4, 8, 16, 32, 64, 1 << 20):
            ops.gemm_wide_set_chunk(chunk)
            out.fill_(float("nan"))
            ops.gemm_bf16x3_wide(a_hi, a_lo, b_hi, b_lo, m, n, k, out)
            e = errs(out, want)
            ms = timed(lambda: ops.gemm_bf16x3_wide(a_hi, a_lo, b_hi, b_lo, m, n, k, out))
            res[f"tc_chunk{chunk if chunk < 1 << 20 else 'inf'}"] = {"max_norm_err": e[0], "elem_err": e[1], "ms": round(ms, 4),
                                                                     "tflops_bf16_issued": round(3 * 2 * m * n * k / ms / 1e9, 1)}
        ops.gemm_wide_set_chunk(16)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
