"""Audiences and the sliced sweep + merge (tests/test_gpu_zz_audience.py) executed on the CPU by the cuemu fiber emulator, at
small shapes: the exact model on both buffer routes and every width, ties and edges, sliced == unsliced from one slice to more
slices than candidates, the merge against a host model, forced slicing of Recommender / SimilarItems, the slice choice, the
one-process row-sharded audience, and Trainer.audience before and after a checkpoint."""
import functools

import pytest

from tests import test_gpu_zz_audience as A
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    lib = harness.emulated_device(monkeypatch)
    from mmssl_b200 import evaluate
    monkeypatch.setattr(evaluate, "Evaluator", functools.partial(evaluate.Evaluator, device="cpu"))
    return lib


@pytest.fixture
def emu_fwd(monkeypatch):
    harness.set_order("fwd")
    lib = harness.emulated_device(monkeypatch)
    from mmssl_b200 import evaluate
    monkeypatch.setattr(evaluate, "Evaluator", functools.partial(evaluate.Evaluator, device="cpu"))
    return lib


@pytest.mark.parametrize("k", [1, 64, 65, 300])
def test_exact_model_both_routes(emu, k):
    A.run_exact(k, U=150, I=12, d=8, device="cpu")


@pytest.mark.parametrize("d", [32, 64, 96, 128, 192, 256])
def test_exact_model_every_width(emu_fwd, d):
    A.run_exact(20 if d % 64 else 70, U=100, I=9, d=d, seed=d, device="cpu")


def test_queries_ties_and_edges(emu_fwd):
    A.run_queries(device="cpu")


@pytest.mark.parametrize("k", [5, 70])
@pytest.mark.parametrize("slices", [1, 2, 3, 7, 301])
def test_sliced_equals_unsliced(emu_fwd, k, slices):
    A.run_sliced(emu_fwd, k, slices, device="cpu")


def test_sliced_equals_unsliced_reversed_threads(emu):
    A.run_sliced(emu, 70, 3, device="cpu")


def test_merge_against_host_model(emu):
    A.run_merge_model(emu, device="cpu")


@pytest.mark.parametrize("slices", [2, 5])
def test_forced_slices_recommend_and_similar(emu_fwd, monkeypatch, slices):
    A.run_forced_slices(monkeypatch, slices, device="cpu")


def test_slice_choice(emu_fwd):
    A.run_slice_choice(device="cpu")


@pytest.mark.parametrize("exclude", ["train", "seen"])
def test_sharded_one_process(emu_fwd, tmp_path, exclude):
    A.run_sharded_one_process(tmp_path, exclude, device="cpu")


def test_trainer_audience(emu_fwd, tmp_path):
    A.run_trainer(tmp_path, device="cpu", epochs=2)


def test_export_and_reader_refusals(emu_fwd, tmp_path):
    """A chunked export reads back as one topk call; each of recommend.read / similar.read / audience.read refuses the other
    two formats."""
    import numpy as np
    import torch
    from mmssl_b200 import audience, recommend, similar
    ua, ia, train = A.problem(40, 30, 32, 3)
    aud = audience.Audience.from_rows(torch.from_numpy(ua), train, {}, {}, 30, 4)
    items = np.array([29, 3, 3, 0, 11, 7, 8], np.int64)
    out = str(tmp_path / "aud")
    assert aud.export(torch.from_numpy(ia), items, out, chunk=3) == items.size
    q, i, s = audience.read(out)
    want_i, want_s = aud.topk(torch.from_numpy(ia), items)
    assert np.array_equal(q, items) and np.array_equal(i, want_i.numpy().astype(np.int32)) and np.array_equal(A._bits(s), A._bits(want_s))
    for reader in (recommend.read, similar.read):
        with pytest.raises(ValueError, match="audience"):
            reader(out)
    rec_out, sim_out = str(tmp_path / "rec"), str(tmp_path / "sim")
    recommend.Recommender.from_rows(torch.from_numpy(ia), train, {}, {}, 40, 4).export(torch.from_numpy(ua), [0, 1], rec_out)
    similar.SimilarItems(torch.from_numpy(ia), 4).export([0, 1], sim_out)
    for o in (rec_out, sim_out):
        with pytest.raises(ValueError, match="not of audiences"):
            audience.read(o)
