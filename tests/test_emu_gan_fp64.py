"""tests/test_gpu_zz_gan_fp64.py executed on the CPU by the cuemu fiber emulator (tests/cuemu) at small sizes: every GAN
kernel and the composite D step / G side against float64, on both GEMM routes and both fiber orders.  The large shapes
(n = 32768, I = 7050) run on the GPU only."""
import pytest

from tests import test_gpu_zz_gan_fp64 as G
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("n,h", [(2, 1), (3, 2), (48, 3), (2, 5), (130, 12), (48, 25), (3, 25)])
def test_bn_ops(emu, n, h):
    G.check_bn_ops(n, h)


@pytest.mark.parametrize("sat", ["none", "high", "low", "half"])
@pytest.mark.parametrize("n,h", [(48, 1), (37, 5), (3, 5)])
def test_head_ops(emu, n, h, sat):
    G.check_head_ops(n, h, sat)


@pytest.mark.parametrize("n,w", [(5, 1), (5, 7), (9, 700)])
def test_gp_rows(emu, n, w):
    G.check_gp_rows(n, w)


def test_usim_and_real_rows(emu):
    G.check_usim_and_real_rows(120, 97, 32, 64)


@pytest.mark.parametrize("n,w", [(2, 1), (7, 33), (64, 97)])
def test_elementwise(emu, n, w):
    G.check_elementwise(n, w)


@pytest.mark.parametrize("route", ["simt", "tc"])
@pytest.mark.parametrize("I,d,B", [(8, 32, 2), (9, 64, 24), (15, 96, 24), (16, 128, 24), (97, 96, 24), (101, 192, 24),
                                   (103, 256, 24), (97, 64, 2)])
def test_d_step_and_g_side(emu, I, d, B, route):
    G.test_d_step_and_g_side_vs_float64(I, d, B, route)


@pytest.mark.parametrize("route", ["simt", "tc"])
@pytest.mark.parametrize("sat", ["all", "half"])
def test_d_step_saturated_heads(emu, sat, route):
    G.test_d_step_saturated_heads(sat, route)


def test_full_step_from_saturated_state_stays_finite(monkeypatch):
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    G.full_step_from_saturated_state("cpu")
