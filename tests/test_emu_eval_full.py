"""Full-mode evaluation (csrc/eval.cu, the kFull instantiation) executed on the CPU by the cuemu fiber emulator through
mmssl_b200/evaluate.py -- the bodies of tests/test_gpu_zz_eval_full.py, in both thread orders."""
import functools

import numpy as np
import pytest

from tests import test_gpu_zz_eval_full as E
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
def test_eval_full_matches_reference_golden(emu, case, split):
    E.test_eval_full_matches_reference_golden(case, split)


def test_eval_full_random_tie_heavy_cases(emu):
    E.test_eval_full_random_tie_heavy_cases()


def test_eval_full_stage_boundary(emu):
    """Positives counts 127..130 and 255..257 (the 128-key shared-memory stage and the power-of-two workspace slots),
    several heavy users in one CTA, users not a multiple of the 8-user tile, duplicate users."""
    rng = np.random.default_rng(11)
    U, I, d, Ks = 11, 700, 8, [5, 20]
    ua = rng.integers(-2, 3, (U, d)).astype(np.float32)
    ia = rng.integers(-2, 3, (I, d)).astype(np.float32)
    train = {u: sorted(rng.choice(I, size=int(rng.integers(1, 200)), replace=False).tolist()) for u in range(U)}
    sizes = [127, 128, 129, 130, 255, 256, 257, 3, 1, 600, 128]
    held = {u: rng.choice(I, size=sizes[u], replace=False).tolist() for u in range(U)}
    ev = E._Ev(train, held, {}, U, I, Ks)
    users = np.array([4, 0, 9, 1, 2, 3, 5, 6, 7, 8, 10, 4, 9], np.int64)
    E.check_against_oracle(ev, ua, ia, users, E._csr(train, U), E._csr(held, U), Ks, False)


def test_eval_full_trainer(emu):
    E.run_trainer_full(device="cpu")
