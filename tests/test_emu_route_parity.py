"""tests/test_gpu_zz_route_parity.py's checks at small sizes on the CPU emulator, in two thread orders.  The 2^21-entry graphs
are too slow here, so the automatic SpMM route is replaced by the explicit impl it resolves to on each side (4 below the
threshold, 16 above); the L2-hint variants (impl 128, 256) run through the model of the cache-hinted loads and stores."""
import pytest
import torch

from tests import test_gpu_zz_route_parity as R
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("impl", [4, 16])
@pytest.mark.parametrize("d,nrhs", [(64, 3), (128, 2), (256, 1)])
def test_spmm_route_sides(emu, impl, d, nrhs):
    R.check_spmm_auto_route(8000, 300, 300, d, nrhs, impl=impl, min_heavy=R.HEAVY_ROW + 1)


@pytest.mark.parametrize("impl", R.VARIANTS)
@pytest.mark.parametrize("d,nrhs", [(64, 3), (128, 2), (256, 1)])
def test_spmm_variant_vs_fp64(emu, impl, d, nrhs):
    R.check_spmm_variant(impl, d, nrhs)


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("n,d", [(1, 64), (2, 128), (63, 64), (64, 128), (65, 64), (127, 128), (128, 64), (129, 64), (129, 128)])
@pytest.mark.parametrize("tau", [0.2, 0.5, 1.0])
def test_infonce_routes(emu, impl, n, d, tau):
    R.check_infonce(n, d, tau, impl)


@pytest.mark.parametrize("n", [70, 200])
def test_infonce_cuda_core_route_d256(emu, n):
    assert not R.check_infonce(n, 256, 0.5, "auto").tc


def test_infonce_blockwise_reference_matches_oracle():
    """The blockwise, checkpointed float64 reference used at n = 16384 equals the oracle's formula."""
    gen = torch.Generator().manual_seed(0)
    t1, t2 = torch.randn(40, 64, generator=gen), torch.randn(40, 64, generator=gen)
    idx = torch.randint(0, 40, (300,), generator=gen)
    t1[idx[5]] = 0
    full = R.infonce_reference(t1, t2, idx, 0.3, 1.7)
    blk = R.infonce_reference(t1, t2, idx, 0.3, 1.7, block=128)
    assert abs(full[0] - blk[0]) < 1e-12 * abs(full[0])
    for a, b in zip(full[1:], blk[1:]):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-12 * float(b.abs().max()))


@pytest.mark.parametrize("n,d", [(128, 64), (129, 128)])
def test_infonce_tc_streams_bitwise(emu, monkeypatch, n, d):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)      # take the side-stream branch (streams are no-ops here)
    R.check_nce_streams_bitwise(n, d)
