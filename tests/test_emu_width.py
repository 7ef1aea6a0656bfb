"""Embedding widths 32, 96 and 192 on the CPU emulator: the bodies of tests/test_gpu_zz_width.py, tests/test_gpu_ops.py and
tests/test_gpu_zz_route_parity.py at small sizes, against float64 or the oracle.  The impl 0 SpMM instances are forced
explicitly (impl 4 below 2^21 edges, impl 16 from there), since a 2^21-entry graph is too slow here."""
import pytest

from tests import test_gpu_ops as T
from tests import test_gpu_zz_proj_grouped as G
from tests import test_gpu_zz_route_parity as R
from tests import test_gpu_zz_width as W
from tests.cuemu import harness

NEW_WIDTHS = W.NEW_WIDTHS


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.fixture
def emu_fwd(monkeypatch):
    harness.set_order("fwd")
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("impl", [4, 16])
@pytest.mark.parametrize("nrhs", [1, 2, 3])
@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_spmm_vs_fp64(emu, d, nrhs, impl):
    """Every epilogue, split and heavy rows (the plan-cut graph), peer stores and bitwise repeatability."""
    R.check_spmm_variant(impl, d, nrhs)


@pytest.mark.parametrize("nrhs", [1, 2, 3])
@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_reduce_rows_epilogue(emu, d, nrhs):
    W.check_reduce_rows(d, nrhs)


@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_rowops(emu, d):
    T.test_rowops_vs_autograd(d)


@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_bpr(emu, d):
    T.test_bpr_fused_and_autograd(d)


@pytest.mark.parametrize("n", [1, 65, 1025])
@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_infonce_cuda_core(emu_fwd, d, n):
    """The ragged last chunk of the d axis: 32 = half a chunk, 96 = one and a half, 192 = three whole chunks."""
    assert not R.check_infonce(n, d, 0.5, "auto").tc


@pytest.mark.parametrize("shapes,max_ctas", [
    ([(300, 32, 640), (130, 32, 70)], 3),       # N = 32: m not a multiple of 128, k not a multiple of 64
    ([(515, 96, 200), (70, 96, 300)], 2),       # N = 96
    ([(130, 192, 70), (200, 192, 130)], 2),     # N = 192
])
def test_projection_group_vs_fp64(emu, shapes, max_ctas):
    G.check_group_vs_fp64(shapes, max_ctas)
    G.check_plan(shapes, max_ctas)
    G.check_group_bitwise_vs_single(shapes, max_ctas)      # the single-problem kernel gives the same partials


@pytest.mark.parametrize("d,modal", [(32, "random"), (96, "random")])
def test_hot_step_vs_oracle(emu_fwd, d, modal):
    W.check_hot_step(d, modal)


def test_rejections(emu_fwd):
    W.check_rejections()


@pytest.mark.parametrize("case", W.WIDTH_CASES)
@pytest.mark.parametrize("proj_impl", ["tc", "simt"])
def test_model_vs_reference_golden(emu_fwd, case, proj_impl):
    """Drop-in Models.MMSSL against the reference's golden vectors; 'simt' takes the CUDA-core projection, whose bias gradient
    (mmssl_colsum) runs 192-thread blocks at d = 96."""
    from tests import test_gpu_model as M
    M.test_model_forward_backward_vs_reference(case, proj_impl)
