"""Recommendations (csrc/eval.cu in its recommendation mode, mmssl_b200/recommend.py) executed on the CPU by the cuemu fiber
emulator: both buffer routes (k <= 64 and k > 64) against a float64 brute force, every supported width, exact ties, short lists,
repeated users, rows of a larger output (ldo > k), bitwise the evaluator's ranked lists, the chunked export, the file logic of
an interrupted export and of ``recommend.read``, and ``Trainer.recommend`` before and after a checkpoint."""
import ctypes as C
import functools
import json
import os

import numpy as np
import pytest
import torch

from mmssl_b200 import recommend
from tests import test_gpu_zz_recommend as R
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
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("k", [1, 64, 65, 300])
def test_lists_both_routes(emu, k):
    R.run_lists(k, device="cpu")


@pytest.mark.parametrize("k", [7, 70])
def test_exact_ties_lower_id_first(emu_fwd, k):
    """Small-integer embeddings and 20 copies of one item row: equal scores, lower item id first, equal to the brute force."""
    R.run_lists(k, U=13, I=260, d=8, kind="ties", seed=4, device="cpu")


@pytest.mark.parametrize("k", [40, 300])
def test_k_above_the_unexcluded_items(emu_fwd, k):
    """120 items, 86 to 99 of them excluded: every list is shorter than k (-1 / 0 padding)."""
    ua, ia, train = R.problem(9, 120, 8, 6, n_excl=(86, 100))
    users = np.arange(9, dtype=np.int64)
    ids, sc = recommend.Recommender.from_rows(torch.from_numpy(ia), train, {}, {}, 9, k).topk(torch.from_numpy(ua), users)
    R.check_lists(ids, sc, ua, ia, users, R._csr(train, 9), k)
    assert (ids[:, -1] == -1).all()


@pytest.mark.parametrize("d", [32, 64, 96, 128, 192, 256])
def test_every_width(emu_fwd, d):
    R.run_lists(65 if d in (96, 256) else 20, U=13, I=200, d=d, seed=d, device="cpu")


def test_rows_of_a_larger_output(emu_fwd):
    """ldo > k: every row of the output keeps its columns past k untouched, on both routes."""
    lib = emu_fwd
    ua, ia, train = R.problem(11, 260, 8, 9)
    ip, ix = R._csr(train, 11)
    users = np.array([3, 1, 4, 1, 5, 9, 2, 6, 5, 3], np.int64)
    for k, ldo in ((10, 17), (70, 75)):
        ids = np.full((users.size, ldo), -7, np.int32)
        sc = np.full((users.size, ldo), 7.0, np.float32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        nb = lib.mmssl_recommend_workspace_bytes(users.size, k, 260, 8)
        ws = np.zeros(max(nb // 8, 1), np.uint64)
        assert lib.mmssl_recommend_topk(p(ua), 8, p(ia), 8, 260, 8, p(users), users.size, p(ip), p(ix), k, ldo, p(ids), p(sc), p(ws),
                                        None) == 0
        assert (ids[:, k:] == -7).all() and (sc[:, k:] == 7.0).all()
        R.check_lists(ids[:, :k].astype(np.int64), sc[:, :k], ua, ia, users, (ip, ix), k)
        assert lib.mmssl_recommend_topk(p(ua), 8, p(ia), 8, 260, 8, p(users), users.size, p(ip), p(ix), k, k - 1, p(ids), p(sc), p(ws),
                                        None) != 0          # ldo < k is refused


@pytest.mark.parametrize("k", [10, 64, 65, 200])
def test_bitwise_evaluator(emu, k):
    R.run_against_evaluator(21, 700, 16, k, 21, device="cpu")


def test_bitwise_evaluator_workspace_slot(emu_fwd):
    """k = 1000, d = 64: the candidate buffers do not fit in shared memory and live in the key_ws slots."""
    assert emu_fwd.mmssl_recommend_workspace_bytes(9, 1000, 1500, 64) > 0
    R.run_against_evaluator(9, 1500, 64, 1000, 9, device="cpu")


def test_empty_user_list_and_bad_ids(emu_fwd):
    ua, ia, train = R.problem(5, 50, 8, 2)
    rec = recommend.Recommender.from_rows(torch.from_numpy(ia), train, {}, {}, 5, 3)
    calls = []
    lib = emu_fwd
    real = recommend._lib.load

    class Spy:
        def __getattr__(self, name):
            calls.append(name)
            return getattr(lib, name)
    recommend._lib.load = lambda require_device=False: Spy()
    try:
        ids, sc = rec.topk(torch.from_numpy(ua), [])
    finally:
        recommend._lib.load = real
    assert ids.shape == (0, 3) and sc.shape == (0, 3) and "mmssl_recommend_topk" not in calls
    for bad in ([0, 5], [-1]):
        with pytest.raises(ValueError, match="outside"):
            rec.topk(torch.from_numpy(ua), bad)
    with pytest.raises(ValueError):
        recommend.Recommender.from_rows(torch.from_numpy(ia), train, {}, {}, 5, 3, exclude="all")


@pytest.mark.parametrize("k", [6, 80])
def test_export_equals_topk(emu_fwd, tmp_path, k):
    R.run_export(tmp_path, k, device="cpu")


def test_export_of_no_user(emu_fwd, tmp_path):
    ua, ia, train = R.problem(5, 50, 8, 2)
    rec = recommend.Recommender.from_rows(torch.from_numpy(ia), train, {}, {}, 5, 3)
    assert rec.export(torch.from_numpy(ua), [], str(tmp_path)) == 0
    u, i, s = recommend.read(str(tmp_path))
    assert u.shape == (0,) and i.shape == (0, 3) and s.shape == (0, 3)


def test_interrupted_export_leaves_no_file(emu_fwd, tmp_path, monkeypatch):
    """An export cut short after its first chunk: no temporary file is left, the files under the final names are the earlier
    export's, unchanged, and nothing is readable -- the earlier export's manifest went when the new export began, so its files
    cannot be read mixed with a half-written set.  Into a fresh directory: nothing at all."""
    rec, uc = R.run_export(tmp_path, 5, device="cpu")
    out = str(tmp_path / "rec")
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
        rec.export(uc, np.arange(20), out, chunk=4)
    assert {f: open(os.path.join(out, f), "rb").read() for f in os.listdir(out)} == data
    with pytest.raises(ValueError, match="no committed"):
        recommend.read(out)
    fresh = str(tmp_path / "fresh")
    n[0] = 0
    with pytest.raises(KeyboardInterrupt):
        rec.export(uc, np.arange(20), fresh, chunk=4)
    assert os.listdir(fresh) == []


def test_failed_file_creation_leaves_no_file(emu_fwd, tmp_path, monkeypatch):
    """open_memmap failing on the second file (a full disk): the first temporary file is removed too."""
    ua, ia, train = R.problem(5, 50, 8, 2)
    rec = recommend.Recommender.from_rows(torch.from_numpy(ia), train, {}, {}, 5, 3)
    real = np.lib.format.open_memmap
    n = [0]

    def full(*a, **k):
        n[0] += 1
        if n[0] == 2:
            raise OSError(28, "No space left on device")
        return real(*a, **k)
    monkeypatch.setattr(np.lib.format, "open_memmap", full)
    with pytest.raises(OSError):
        rec.export(torch.from_numpy(ua), [0, 1], str(tmp_path))
    assert os.listdir(tmp_path) == []


def test_exclusion_rows_checked(emu_fwd):
    """The exclusion CSR must be on the item table's device and sorted within each row (the kernel binary-searches it)."""
    ua, ia = torch.zeros(3, 8), torch.zeros(10, 8)
    ip, ix = torch.tensor([0, 2, 2, 4]), torch.tensor([5, 1, 2, 3])
    with pytest.raises(ValueError, match="sorted"):
        recommend.Recommender(ia, (ip, ix), 3)
    ok = torch.tensor([1, 5, 2, 3])                               # a row may start below the previous row's last item
    recommend.Recommender(ia, (ip, ok), 3)
    with pytest.raises(ValueError, match="the item table on"):
        recommend.Recommender(ia, (ip.to("meta"), ok.to("meta")), 3)
    with pytest.raises(TypeError):
        recommend.Recommender(ia, (ip.int(), ok), 3)


def _save_rank(d, r, w, u, export_id, manifest=True):
    for f, a in (("users", u.astype(np.int64)), ("ids", np.stack([u, u]).T.astype(np.int32)),
                 ("scores", np.stack([u, -u]).T.astype(np.float32))):
        np.save(os.path.join(d, f"rank{r:05d}-of-{w:05d}.{f}.npy"), a)
    if manifest:
        with open(os.path.join(d, f"rank{r:05d}-of-{w:05d}.json"), "w") as fh:
            json.dump(dict(format="mmssl_b200.recommend.v1", export=export_id, n=int(u.size), k=2), fh)


def test_read_checks_the_rank_files(tmp_path):
    """Pure file logic: committed rank files concatenated in user order; a missing rank manifest, rank files of different
    exports, exports of two world sizes, both layouts at once, or a manifest naming other shapes are refused."""
    d = str(tmp_path)
    rows = {0: np.array([1, 0, 2]), 1: np.array([5, 3])}
    for r, u in rows.items():
        _save_rank(d, r, 2, u, 9)
    u, i, s = recommend.read(d)
    assert u.tolist() == [0, 1, 2, 3, 5] and i[:, 0].tolist() == [0, 1, 2, 3, 5] and s[:, 1].tolist() == [0, -1, -2, -3, -5]
    _save_rank(d, 1, 2, rows[1], 10)
    with pytest.raises(ValueError, match="different exports"):
        recommend.read(d)
    _save_rank(d, 1, 2, rows[1], 9)
    _save_rank(d, 0, 3, np.zeros(0, np.int64), 4)
    with pytest.raises(ValueError, match="several world sizes"):
        recommend.read(d)
    os.remove(os.path.join(d, "rank00000-of-00003.json"))
    _save_rank(d, 1, 2, rows[1], 9, manifest=False)
    os.remove(os.path.join(d, "rank00001-of-00002.json"))
    with pytest.raises(ValueError, match="world size 2 is incomplete"):
        recommend.read(d)
    _save_rank(d, 1, 2, np.array([5, 3, 4]), 9, manifest=False)
    with open(os.path.join(d, "rank00001-of-00002.json"), "w") as fh:
        json.dump(dict(format="mmssl_b200.recommend.v1", export=9, n=2, k=2), fh)
    with pytest.raises(ValueError, match="shapes"):
        recommend.read(d)
    with open(os.path.join(d, "manifest.json"), "w") as fh:
        json.dump({}, fh)
    with pytest.raises(ValueError, match="one-GPU and a row-sharded"):
        recommend.read(d)
    with pytest.raises(ValueError, match="no committed"):
        recommend.read(str(tmp_path / "nothing"))


def test_union_csr():
    a = (np.array([0, 2, 2, 3]), np.array([4, 1, 0]))
    b = (np.array([0, 1, 3, 3]), np.array([1, 7, 2], np.int32))
    ip, ix = recommend.union_csr(a, b)
    assert ip.tolist() == [0, 2, 4, 5] and ix.tolist() == [1, 4, 2, 7, 0]
    seen = recommend.exclusion_rows({0: [3, 1]}, {0: [1, 9], 2: [4]}, {1: [0]}, "seen")
    assert seen == {0: [1, 3, 9], 1: [0], 2: [4]}


@pytest.mark.parametrize("exclude", ["train", "seen"])
def test_sharded_one_process(emu_fwd, tmp_path, exclude):
    R.run_sharded_one_process(tmp_path, exclude, device="cpu")


def test_trainer_recommend(emu_fwd, tmp_path):
    R.run_trainer(tmp_path, device="cpu")
