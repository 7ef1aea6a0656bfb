"""tools/recommend.py --fold-in end to end on the CPU emulator: a Trainer run on tests/golden/dataset_small saves its checkpoint, the
tool rebuilds the Trainer from it and exports the lists of the queries of an .npz file (id and new-user rows, an empty row,
duplicates); the files read back with ``foldin.read`` equal ``Trainer.recommend_for`` of the saved run, for both exclusion sets, a
file without ``users`` folds every row as a new user, and --fold-in together with --audience is refused.  (The row-sharded mode
runs in tests/test_dist_emu_foldin.py.)"""
import os
import runpy
import sys

import numpy as np
import pytest
import torch

from tests.cuemu import harness
from tests.test_gpu_zz_recommend import GOLD, _bits, trainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("exclude", ["train", "seen"])
def test_foldin_tool_on_a_trainer_checkpoint(monkeypatch, tmp_path, capsys, exclude):
    from mmssl_b200 import foldin, recommend
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    from mmssl_b200.dataset import ReferenceDataset
    real = ReferenceDataset.load.__func__
    monkeypatch.setattr(ReferenceDataset, "load", classmethod(lambda cls, path, mmap_features=True: real(cls, path, False)))
    ckpt = str(tmp_path / "run.ckpt")
    tr = trainer("cpu", epochs=1, ckpt=ckpt)
    tr.train()
    I = tr.n_items
    ip = np.array([0, 3, 3, 9, 10, 12], np.int64)
    ix = np.array([4, 1, 4, 0, 2, 5, 7, 9, 9, I - 1, 3, 8], np.int64)
    users = np.array([2, -1, 7, -1, tr.n_users - 1], np.int64)
    with_users, no_users = str(tmp_path / "q.npz"), str(tmp_path / "q_new.npz")
    np.savez(with_users, indptr=ip, indices=ix, users=users)
    np.savez(no_users, indptr=ip, indices=ix)

    def run(out, *extra):
        monkeypatch.setattr(sys, "argv", ["recommend.py", os.path.join(GOLD, "dataset_small"), "--checkpoint", ckpt, "--k", "6",
                                          "--exclude", exclude, "--out", out, "--chunk", "2", *extra])
        runpy.run_path(os.path.join(ROOT, "tools", "recommend.py"), run_name="__main__")
        return capsys.readouterr().out

    for name, path, us in (("ids", with_users, users), ("new", no_users, None)):
        out = str(tmp_path / name)
        assert '"queries": 5' in run(out, "--fold-in", path)
        assert sorted(os.listdir(out)) == ["ids.npy", "manifest.json", "queries.npy", "scores.npy"]
        q, i, s = foldin.read(out)
        want_ids, want_sc = tr.recommend_for((ip, ix), 6, us, exclude)
        assert np.array_equal(q, np.arange(5)) and np.array_equal(i, want_ids.numpy().astype(np.int32))
        assert np.array_equal(_bits(s), _bits(want_sc))
        with pytest.raises(ValueError, match="fold-in"):
            recommend.read(out)
    with pytest.raises(SystemExit):
        run(str(tmp_path / "bad"), "--fold-in", with_users, "--audience")
