"""Evaluation with wide cut-off lists (csrc/eval.cu, eval_wide_kernel) executed on the CPU by the cuemu fiber emulator
through mmssl_b200/evaluate.py -- the bodies of tests/test_gpu_zz_eval_wide.py, in both thread orders, plus sizes that
force many compactions of a shared-memory buffer, a global workspace slot, and max(Ks) >= n_items."""
import functools

import numpy as np
import pytest

from tests import test_gpu_zz_eval_wide as E
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    lib = harness.emulated_device(monkeypatch)
    from mmssl_b200 import evaluate
    monkeypatch.setattr(evaluate, "Evaluator", functools.partial(evaluate.Evaluator, device="cpu"))
    return lib


@pytest.mark.parametrize("case", E.CASES)
@pytest.mark.parametrize("split", ["test", "val"])
def test_eval_wide_matches_reference_golden(emu, case, split):
    E.test_eval_wide_matches_reference_golden(case, split)


@pytest.mark.parametrize("Ks,flag,slot", [
    ([70, 5, 100, 65], "part", False),        # cap 512 in shared memory: a compaction every few sweeps
    ([800, 10], "full", True),                # cap 1920: 123 KiB per CTA -> a global workspace slot, compactions there
    ([3000, 7, 64, 1], "part", True),         # max(Ks) == n_items: every candidate kept, sorted in the slot
    ([4000] + list(range(1, 12)), "full", True),   # max(Ks) > n_items, 12 cut-offs
])
def test_eval_wide_compactions_and_workspace(emu, Ks, flag, slot):
    """Scores increasing along the item axis (every sweep appends: the worst case for the threshold filter), users not a
    multiple of the 8-user tile, an empty training row, duplicate users, held-out rows longer than the 128-key stage."""
    rng = np.random.default_rng(len(Ks))
    U, I, d = 11, 3000, 8
    ua = np.abs(rng.standard_normal((U, d))).astype(np.float32)
    ia = (np.abs(rng.standard_normal((I, d))) * np.linspace(0.1, 3.0, I)[:, None]).astype(np.float32)
    train = {u: sorted(rng.choice(I, size=int(rng.integers(0, 400)), replace=False).tolist()) for u in range(U)}
    train[3] = []
    train = {u: v for u, v in train.items() if v}
    held = {u: rng.choice(I, size=int(rng.choice([rng.integers(1, 30), rng.integers(130, 300)])), replace=False).tolist()
            for u in range(U)}
    assert (emu.mmssl_eval_wide_workspace_bytes(U, max(Ks), I, d) > 0) == slot
    ev = E._Ev(train, held, {}, U, I, Ks, test_flag=flag)
    users = np.array([4, 0, 9, 1, 2, 3, 5, 6, 7, 8, 10, 4], np.int64)
    E.check_against_oracle(ev, ua, ia, users, E._csr(train, U), E._csr(held, U), Ks, False)


def test_eval_wide_tie_heavy(emu):
    """Small-integer embeddings: many exactly equal scores, so equal scores must keep the lower item id first through the
    radix select and sort."""
    rng = np.random.default_rng(77)
    U, I, d, Ks = 13, 900, 4, [65, 300, 10, 65]
    ua = rng.integers(-2, 3, (U, d)).astype(np.float32)
    ia = rng.integers(-2, 3, (I, d)).astype(np.float32)
    train = {u: sorted(rng.choice(I, size=int(rng.integers(1, 300)), replace=False).tolist()) for u in range(U)}
    held = {u: rng.choice(I, size=int(rng.integers(1, 40)), replace=False).tolist() for u in range(U)}
    ev = E._Ev(train, held, {}, U, I, Ks, test_flag="full")
    E.check_against_oracle(ev, ua, ia, rng.permutation(U).astype(np.int64), E._csr(train, U), E._csr(held, U), Ks, False)


def test_eval_wide_consistent_with_narrow(emu):
    E.run_consistency_with_narrow(U=20, I=700, d=8, full=True)


def test_eval_wide_trainer(emu):
    E.run_trainer_wide(device="cpu")


def test_eval_wide_rejected_input(emu):
    E.run_rejected_input(device="cpu")
