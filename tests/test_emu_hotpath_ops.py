"""Kernels of the hot path that are parity-green on a real H100 (tests/test_gpu_ops.py), executed on the CPU by
the cuemu fiber emulator through the same bodies.  Two purposes: (1) cross-check the emulator itself against kernels
whose GPU behaviour is known -- warp-group shuffles, block reductions, 128-bit vector atomics, last-arriver counters;
(2) keep these kernels under test in the `-m "not gpu"` suite, which runs where there is no GPU."""
import pytest

from tests import test_gpu_ops as T
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("ta,tb", [(False, False), (True, True)])
def test_sgemm(emu, ta, tb):
    T.test_sgemm(ta, tb)


@pytest.mark.parametrize("d", [64, 128, 256])
def test_rowops(emu, d):
    T.test_rowops_vs_autograd(d)


@pytest.mark.parametrize("d", [64, 128])
def test_bpr(emu, d):
    T.test_bpr_fused_and_autograd(d)


@pytest.mark.parametrize("n,d", [(64, 64), (257, 64), (130, 128), (96, 256), (1500, 64)])
def test_infonce(emu, n, d):
    T.test_infonce_forward_backward(n, d)


def test_feat_reg_and_adamw(emu):
    T.test_feat_reg_autograd()
    T.test_adamw_matches_torch()


def test_sampler(emu):
    T.test_device_triple_sampler_semantics()


@pytest.mark.parametrize("shape_nnz", [((50, 70), 400), ((1, 1), 1), ((300, 200), 0), ((2000, 900), 60000)])
def test_csr_from_coo(emu, shape_nnz):
    T.test_csr_from_coo(shape_nnz)


def test_row_normalize(emu):
    T.test_row_normalize_matches_reference_formula()


@pytest.mark.parametrize("d,nrhs", [(64, 1), (64, 3), (128, 2), (256, 1)])
def test_spmm_plain(emu, d, nrhs):
    T.test_spmm_plain(d, nrhs)


@pytest.mark.parametrize("impl,nrhs", [(2, 1), (4, 3), (6, 1)])
def test_spmm_impl_variants(emu, impl, nrhs):
    T.test_spmm_impl_variants(impl, nrhs)


def test_spmm_empty_and_epilogues(emu):
    T.test_spmm_empty_and_tiny()
    T.test_spmm_epilogues(64)


@pytest.mark.parametrize("d,nrhs,base_impl", [(64, 1, 4), (64, 2, 16), (128, 1, 16), (128, 2, 4), (256, 1, 4), (64, 3, 4)])
def test_spmm_early_prefetch_variant(emu, d, nrhs, base_impl):
    from tests import test_gpu_zz_more_ops as Z
    Z.test_spmm_early_prefetch_variant_matches_default(d, nrhs, base_impl)


@pytest.mark.parametrize("d,nrhs,blocks,pre", [(64, 1, 0, 0), (64, 1, 7, 64), (64, 2, 5, 0), (128, 1, 3, 64), (128, 2, 11, 0), (256, 1, 2, 64), (64, 3, 4, 0)])
def test_spmm_pipelined_walk(emu, d, nrhs, blocks, pre):
    from tests import test_gpu_zz_more_ops as Z
    Z.test_spmm_pipelined_walk_matches_default(d, nrhs, blocks, pre)


@pytest.mark.parametrize("cuts,d,nrhs", [((16, 8, 64, 16), 64, 1), ((32, 16, 1024, 64), 128, 2), ((24, 24, 48, 5), 256, 1), ((16, 8, 64, 16), 128, 2)])
def test_spmm_plan_cuts(emu, cuts, d, nrhs):
    from tests import test_gpu_zz_more_ops as Z
    Z.test_spmm_plan_cuts(cuts, d, nrhs)


@pytest.mark.parametrize("n,d,two", [(777, 64, False), (777, 128, True), (100100, 64, True)])
def test_id_fuse2_against_autograd(emu, n, d, two):
    from tests import test_gpu_zz_more_ops as Z
    Z.test_id_fuse2_against_autograd(n, d, two)


@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
def test_sgemm_large_tiles(emu, ta, tb):
    from tests import test_gpu_zz_more_ops as Z
    Z.test_sgemm_large_tiles(ta, tb, 300, 700, 130)
    Z.test_sgemm_large_tiles(ta, tb, 128, 512, 8)


@pytest.mark.parametrize("d", [64, 128])
def test_spmm_length_sorted_work_items(emu, monkeypatch, d):
    from tests import test_gpu_zz_more_ops as Z
    Z.test_spmm_length_sorted_work_items(d, monkeypatch)
