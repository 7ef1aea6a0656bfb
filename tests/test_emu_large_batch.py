"""The multi-CTA device sampler (csrc/sampler.cu) executed on the CPU by the cuemu emulator, in both thread orders: the bodies
of tests/test_gpu_zz_large_batch.py at small n_exist, with several select blocks, every batch size class (one triple, ragged,
n_exist - 1, a full permutation, with replacement) and the sampler class's routing above 1024 triples."""
import pytest

from tests import test_gpu_zz_large_batch as L
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


def test_multi_sampler_semantics_small(emu):
    csr = L.random_csr(300, 40, seed=1)        # 257 eligible users: two select blocks
    n_exist = int((csr.indptr[1:] > csr.indptr[:-1]).sum())
    L.check_multi_semantics(csr, [1, 7, 100, 256, n_exist - 1, n_exist, n_exist + 1, 700])


def test_multi_sampler_routing_above_1024(emu):
    csr = L.random_csr(1400, 60, seed=2)       # 1200 eligible users
    L.check_class_routing(csr, 1100)           # distinct
    L.check_class_routing(csr, 1500)           # with replacement
