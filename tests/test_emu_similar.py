"""Similar items (mmssl_unit_rows in csrc/rowops.cu, the ranking sweep of csrc/eval.cu, mmssl_b200/similar.py) executed on the CPU by
the cuemu fiber emulator: the unit rows at every width, exact lists on both buffer routes (k <= 64 and k > 64) and with k >= n_items,
random tables in the three spaces against float64, feature queries, the chunked export and its file logic, both ranks of a
row-sharded export in one process, and ``Trainer.similar_items`` before and after a checkpoint."""
import os

import numpy as np
import pytest
import torch

from mmssl_b200 import recommend, similar
from tests import test_gpu_zz_similar as S
from tests.cuemu import harness


@pytest.fixture
def emu(monkeypatch):
    harness.set_order("fwd")
    return harness.emulated_device(monkeypatch)


@pytest.fixture(params=["fwd", "rev"])
def emu_both(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("d", S.WIDTHS)
def test_unit_rows(emu_both, d):
    S.run_unit_rows(d, device="cpu")


@pytest.mark.parametrize("k", [1, 64, 65, 150, 400])
def test_exact_lists(emu, k):
    """k = 1, both routes, k = n_items and k > n_items: the lists are the float64 brute force's, ties lower id first."""
    S.run_exact(k, n=150, d=32, device="cpu")


@pytest.mark.parametrize("space", ["model", "image", "text"])
@pytest.mark.parametrize("k", [20, 100])
def test_random_tables(emu, space, k):
    S.run_random(230, 32, k, space, 40, device="cpu")


@pytest.mark.parametrize("space", ["image", "text"])
def test_feature_queries(emu, space):
    S.run_features(230, 32, 12, space, device="cpu")


@pytest.mark.parametrize("k", [6, 80])
def test_export_equals_topk(emu, tmp_path, k):
    S.run_export(tmp_path, k, device="cpu")


def test_checks(emu):
    t = torch.randn(10, 32)
    with pytest.raises(ValueError, match="space"):
        similar.SimilarItems(t, 3, "audio")
    with pytest.raises(ValueError, match="k must be"):
        similar.SimilarItems(t, 0)
    sim = similar.SimilarItems(t, 3)
    for bad in ([0, 10], [-1]):
        with pytest.raises(ValueError, match="outside"):
            sim.topk(bad)
    ids, sc = sim.topk([])
    assert ids.shape == (0, 3) and sc.shape == (0, 3)
    with pytest.raises(ValueError, match="image"):
        sim.topk_features(np.zeros((1, 4), np.float32), np.zeros((1, 4), np.float32))
    with pytest.raises(ValueError, match="block"):
        similar.ShardedSimilarItems(similar.RowPartition(10, 2), 0, 3).topk(t, [0])


def test_wrong_feature_widths_write_nothing(emu, tmp_path):
    """export_features of rows of the wrong width is refused before anything is written."""
    sim = S.run_features(60, 32, 5, "image", device="cpu", Dv=24, Dt=16)
    out = str(tmp_path / "feat")
    with pytest.raises(ValueError, match="image 24 / text 16"):
        sim.export_features(np.zeros((3, 20), np.float32), np.zeros((3, 16), np.float32), out)
    assert not os.path.exists(out)


def test_sharded_table_of_any_layout(emu):
    """A rank's block given as a strided view (here the transpose of a transposed copy, and a column slice of a wider buffer)
    ranks like its contiguous copy; a table that is not fp32 is refused."""
    from mmssl_b200.parallel import RowPartition
    t = torch.randn(21, 32)
    pi = RowPartition(21, 2)
    block = pi.local(t, 1)
    wide = torch.zeros(pi.block, 40)
    wide[:, 3:35] = block
    sh = similar.ShardedSimilarItems(pi, 1, 4, device="cpu")
    sh.gather = lambda unit_local: similar.ops.unit_rows(t)
    want_i, want_s, _ = sh.topk(block, np.arange(21))
    for view in (block.t().contiguous().t(), wide[:, 3:35]):
        got_i, got_s, _ = sh.topk(view, np.arange(21))
        assert torch.equal(got_i, want_i) and torch.equal(got_s, want_s)
    with pytest.raises(TypeError, match="fp32"):
        sh.topk(block.double(), np.arange(21))


def test_interrupted_export_is_not_readable(emu, tmp_path, monkeypatch):
    """An export cut short after its first chunk leaves no temporary file and nothing readable (the earlier export's manifest
    went when the new one began); a file set without its manifest is refused."""
    sim = S.run_export(tmp_path, 5, device="cpu")
    out = str(tmp_path / "sim")
    data = {f: open(os.path.join(out, f), "rb").read() for f in os.listdir(out) if f.endswith(".npy")}
    real = recommend.Recommender._launch
    n = [0]

    def cut(self, *a):
        n[0] += 1
        if n[0] == 2:
            raise KeyboardInterrupt
        return real(self, *a)
    monkeypatch.setattr(recommend.Recommender, "_launch", cut)
    with pytest.raises(KeyboardInterrupt):
        sim.export(np.arange(20), out, chunk=4)
    assert {f: open(os.path.join(out, f), "rb").read() for f in os.listdir(out)} == data
    with pytest.raises(ValueError, match="no committed similar-items"):
        similar.read(out)
    fresh = str(tmp_path / "fresh")
    n[0] = 0
    with pytest.raises(KeyboardInterrupt):
        sim.export(np.arange(20), fresh, chunk=4)
    assert os.listdir(fresh) == []


def test_rank_files_of_the_other_kind_are_refused(emu, tmp_path):
    """Row-sharded layouts: a similar-items rank set is refused by recommend.read and the other way round; a similar-items set
    without a rank's manifest is incomplete."""
    from mmssl_b200.parallel import RowPartition
    t = torch.randn(21, 32)
    pi = RowPartition(21, 2)
    out = str(tmp_path / "sh")
    for r in range(2):
        sh = similar.ShardedSimilarItems(pi, r, 4, "image", device="cpu")
        sh.gather = lambda unit_local: similar.ops.unit_rows(t)
        sh.export_id = lambda: 99
        sh.export(pi.local(t, r), np.arange(21), out)
    items, ids, _ = similar.read(out)
    assert items.tolist() == list(range(21)) and ids.shape == (21, 4)
    with pytest.raises(ValueError, match="similar items"):
        recommend.read(out)
    os.remove(os.path.join(out, "rank00001-of-00002.json"))
    with pytest.raises(ValueError, match="incomplete"):
        similar.read(out)


def test_sharded_one_process(emu, tmp_path):
    S.run_sharded_one_process(tmp_path, device="cpu")


def test_trainer_similar_items(emu, tmp_path):
    S.run_trainer(tmp_path, device="cpu")
