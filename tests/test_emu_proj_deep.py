"""The deep-ring instance of the grouped projection GEMM (csrc/proj_tc.cu) executed on the CPU by the cuemu PTX model, in both
thread orders: the bodies of tests/test_gpu_zz_proj_deep.py at small sizes.  A grid of at most one CTA per SM selects the
deep instance at N = 32 / 64; with a few CTAs and short K slices every CTA walks several units and the 4- / 5-stage ring
wraps its mbarrier phases inside and across units."""
import pytest

from tests import test_gpu_zz_proj_deep as D
from tests import test_gpu_zz_proj_grouped as G
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("shapes,max_ctas", [
    ([(300, 32, 640), (300, 32, 128)], 3),      # N = 32: 5 stages, units of 10 and 2 k-blocks
    ([(515, 64, 200), (130, 64, 70)], 2),       # ragged M and K
    ([(256, 64, 3200)], 2),                     # one problem, more than kMaxChainKb k-blocks
    ([(200, 128, 130), (70, 128, 300)], 3),     # N = 128: the one instance
    ([(300, 64, 640), (300, 64, 128)], 132),    # the engine's cap: one unit per CTA
])
def test_deep_vs_fp64(emu, shapes, max_ctas):
    G.check_group_vs_fp64(shapes, max_ctas)
    G.check_plan(shapes, max_ctas)


@pytest.mark.parametrize("shapes,max_ctas", [
    ([(300, 32, 640), (300, 32, 128)], 3),
    ([(515, 64, 200), (130, 64, 70)], 2),
    ([(300, 64, 640), (300, 64, 128)], 132),
])
def test_deep_bitwise_vs_single_kernel(emu, shapes, max_ctas):
    G.check_group_bitwise_vs_single(shapes, max_ctas)


@pytest.mark.parametrize("shapes", D.SHAPES, ids=D.IDS)
def test_deep_plan_at_full_size(emu, shapes):
    """Host-side plans of the benchmark's shapes at the 132-CTA cap (no kernel runs)."""
    G.check_plan(shapes, D.CAP)


def test_hot_step_draws_the_same_masks(emu):
    D.test_hot_step_draws_the_same_masks()
