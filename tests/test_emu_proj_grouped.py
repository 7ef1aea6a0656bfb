"""The grouped, persistent projection GEMM (csrc/proj_tc.cu) executed on the CPU by the cuemu PTX model, in both thread
orders: the bodies of tests/test_gpu_zz_proj_grouped.py at small sizes, with the grid capped to a few CTAs so that every
CTA walks several units and the TMA / mbarrier ring carries its phases across unit boundaries."""
import pytest

from tests import test_gpu_zz_proj_grouped as G
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("shapes,max_ctas", [
    ([(300, 64, 640), (300, 64, 128)], 3),      # forward-like: a long and a short K, split-K on both
    ([(515, 64, 200), (130, 64, 70)], 2),       # ragged M and K (not multiples of 128 / 64)
    ([(256, 64, 3200)], 2),                     # one problem; 50 k-blocks: more than kMaxChainKb, so at least two slices
    ([(200, 128, 130), (70, 128, 300)], 3),     # N = 128
    ([(130, 256, 70), (64, 256, 64)], 2),       # N = 256
])
def test_group_vs_fp64(emu, shapes, max_ctas):
    G.check_group_vs_fp64(shapes, max_ctas)
    G.check_plan(shapes, max_ctas)


@pytest.mark.parametrize("shapes,max_ctas", [
    ([(300, 64, 640), (300, 64, 128)], 3),
    ([(515, 64, 200), (130, 64, 70)], 2),
])
def test_group_bitwise_vs_single_kernel(emu, shapes, max_ctas):
    G.check_group_bitwise_vs_single(shapes, max_ctas)


@pytest.mark.parametrize("shapes", [G.BABY_FWD, G.BABY_WGRAD, G.SPORTS_FWD, G.SPORTS_WGRAD])
def test_plan_at_full_size(emu, shapes):
    """Host-side plans of the benchmark's shapes (no kernel runs)."""
    G.check_plan(shapes)


def test_baby_forward_keeps_the_single_kernel_slices(emu):
    G.test_baby_forward_keeps_the_single_kernel_slices()
