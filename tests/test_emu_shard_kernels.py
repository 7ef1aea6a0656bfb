"""tests/test_gpu_zz_shard_kernels.py executed on the CPU by the cuemu fiber emulator (tests/cuemu): gather_owned and
scatter_add_owned at every width, edge ids, lo == hi and n = 0, in both fiber orders."""
import pytest

from tests import test_gpu_zz_shard_kernels as G
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("d", G.WIDTHS)
@pytest.mark.parametrize("lo,hi", G.BLOCKS)
def test_gather_owned(emu, d, lo, hi):
    G.check_gather_owned(d, lo, hi)


@pytest.mark.parametrize("d", G.WIDTHS)
@pytest.mark.parametrize("lo,hi", G.BLOCKS)
def test_scatter_add_owned(emu, d, lo, hi):
    G.check_scatter_add_owned(d, lo, hi)


@pytest.mark.parametrize("d", [4, 96])
def test_empty_batch(emu, d):
    G.check_gather_owned(d, 20, 37, n=0)
    G.check_scatter_add_owned(d, 20, 37, n=0)
