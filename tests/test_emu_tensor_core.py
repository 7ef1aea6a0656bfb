"""The wgmma / TMA kernels executed on the CPU through cuemu's functional model of the PTX they issue (tests/cuemu/cuemu_ptx.cpp:
mbarrier phases and transaction counts, 2-D TMA box copies with out-of-bounds zero fill and the 128-byte swizzle, UMMA
shared-memory descriptors, wgmma accumulator fragments).

  * calibration: csrc/proj_tc.cu -- parity-green on the H100 -- computes the right products through the model, for its three
    tile widths, with split-K, ragged M and K;
  * csrc/gemm_wide.cu -- written without GPU access, shares tc_common.cuh's descriptor / swizzle / pipeline helpers with the
    kernel above -- is then checked in what is its own: tiling over N, out-of-bounds rows and columns, the alpha / accumulate
    epilogue with vector and scalar stores.
The model proves protocol and indexing logic, not timing or true asynchrony; the GPU test of gemm_wide.cu stays gated."""
import pytest

from tests.cuemu import harness


@pytest.fixture
def emu(monkeypatch):
    harness.set_order("fwd")
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("m,n,k", [(300, 64, 96), (200, 128, 130), (130, 256, 70), (515, 64, 200)])
def test_projection_gemm_kernel_through_the_ptx_model(emu, m, n, k):
    from tests import test_gpu_ops as T
    T.test_gemm_bf16x3_tensor_core(m, n, k)


@pytest.mark.parametrize("m,n,k", [(64, 24, 96), (300, 200, 96), (130, 257, 70), (5, 1, 8), (260, 600, 200)])
def test_wide_gemm_kernel_through_the_ptx_model(emu, monkeypatch, m, n, k):
    from tests import test_gpu_zzz_gemm_wide as W
    W.test_gemm_wide_vs_fp64(m, n, k)


@pytest.mark.parametrize("chunk", [1, 2, 3])
@pytest.mark.parametrize("m,n,k", [(130, 257, 200), (64, 24, 330)])
def test_wide_gemm_multi_pass_accumulation(emu, chunk, m, n, k):
    """The K range cut into several accumulation passes (the epilogue folds each pass into C): same result."""
    from mmssl_b200 import ops
    from tests import test_gpu_zzz_gemm_wide as W
    ops.gemm_wide_set_chunk(chunk)
    try:
        W.test_gemm_wide_vs_fp64(m, n, k)
    finally:
        ops.gemm_wide_set_chunk(16)


def test_model_rejects_what_the_hardware_would_not_run(emu):
    """The driver-side checks of the tensor-map encoder the model re-states: strides and base 16-byte aligned."""
    import torch
    from mmssl_b200 import _lib, ops
    a = torch.randn(16, 64)
    hi, lo = ops.split_bf16(a)
    out = torch.empty(16, 16)
    with pytest.raises(_lib.MmsslLibraryError):                  # leading dimension not a multiple of 8 elements
        lib = _lib.load()
        _lib.check(lib.mmssl_gemm_bf16x3_wide(_lib.ptr(hi), _lib.ptr(lo), 60, _lib.ptr(hi), _lib.ptr(lo), 64, 16, 16, 60, 1.0, 0,
                                              _lib.ptr(out), 16, _lib.stream()))
