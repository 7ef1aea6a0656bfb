"""Fold-in (tests/test_gpu_zz_foldin.py) executed on the CPU by the cuemu fiber emulator, at small shapes: float64 bounds at every
width with rows on both sides of each SpMM cut, bitwise identity with the forward with empty and non-empty modality graphs, batch
invariance, semantics and exports, the one-process world-2 ShardedFoldIn, and the Trainer (recommend_for == recommend, after a
checkpoint reload, and the next training step untouched)."""
import functools

import pytest

from tests import test_gpu_zz_foldin as F
from tests.cuemu import harness


@pytest.fixture
def emu(monkeypatch):
    harness.set_order("fwd")
    lib = harness.emulated_device(monkeypatch)
    from mmssl_b200 import evaluate
    monkeypatch.setattr(evaluate, "Evaluator", functools.partial(evaluate.Evaluator, device="cpu"))
    return lib


@pytest.fixture(params=["rev", "shuffle:3"])
def emu_order(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("d,K", [(32, 1), (64, 2), (96, 3), (128, 1), (192, 2), (256, 3)])
def test_against_float64(emu, d, K):
    F.run_fp64(d, K, I=1200, degs=(0, 1, 63, 64, 65, 1024, 1025, 1200), U=6, device="cpu")


def test_against_float64_thread_orders(emu_order):
    F.run_fp64(64, 2, I=300, degs=(0, 1, 64, 65, 300), U=4, device="cpu")


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("d,K", [(64, 2), (96, 1), (128, 3)])
def test_identity_with_forward(emu, d, K, fused):
    F.run_identity(d, K, fused, U=24, I=1600, device="cpu")


def test_batch_invariance_and_determinism(emu):
    F.run_invariance(n_others=300, device="cpu")


def test_semantics(emu, tmp_path):
    F.run_semantics(tmp_path, device="cpu")


def test_sharded_one_process(emu):
    F.run_sharded_one_process(device="cpu")


def test_trainer(emu, tmp_path):
    F.run_trainer(tmp_path, device="cpu")
