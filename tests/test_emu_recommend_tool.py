"""tools/recommend.py end to end on the CPU emulator: a Trainer run on tests/golden/dataset_small saves its checkpoint, the tool
rebuilds the Trainer from the checkpoint and the dataset directory and exports every user's list; the files are readable with
``recommend.read`` and equal to ``Trainer.recommend`` of the saved run, for both exclusion sets.  (The tool itself only runs on
GPUs; a typo in it costs GPU-minutes.)"""
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
def test_recommend_tool_on_a_trainer_checkpoint(monkeypatch, tmp_path, capsys, exclude):
    """A run trained at id_cat_rate / model_cat_rate other than the defaults (neither is in the checkpoint): with the run's rates
    the tool writes Trainer.recommend's lists bit for bit; with the defaults it writes other lists."""
    from mmssl_b200 import recommend
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    # the emulated .to("cuda") does not copy: the model's feature tables would stay on the loader's read-only maps
    from mmssl_b200.dataset import ReferenceDataset
    real = ReferenceDataset.load.__func__
    monkeypatch.setattr(ReferenceDataset, "load", classmethod(lambda cls, path, mmap_features=True: real(cls, path, False)))
    ckpt = str(tmp_path / "run.ckpt")
    tr = trainer("cpu", epochs=1, ckpt=ckpt, id_cat_rate=0.2, model_cat_rate=0.7)
    tr.train()
    want_ids, want_sc = tr.recommend(np.arange(tr.n_users), 7, exclude)

    def run(out, *rates):
        monkeypatch.setattr(sys, "argv", ["recommend.py", os.path.join(GOLD, "dataset_small"), "--checkpoint", ckpt, "--k", "7",
                                          "--exclude", exclude, "--out", out, "--chunk", "5", *rates])
        runpy.run_path(os.path.join(ROOT, "tools", "recommend.py"), run_name="__main__")
        assert '"users": %d' % tr.n_users in capsys.readouterr().out
        return recommend.read(out)

    out = str(tmp_path / "out")
    u, i, s = run(out, "--id-cat-rate", "0.2", "--model-cat-rate", "0.7")
    assert sorted(os.listdir(out)) == ["ids.npy", "manifest.json", "scores.npy", "users.npy"]
    assert np.array_equal(u, np.arange(tr.n_users))
    assert np.array_equal(i, want_ids.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(want_sc))
    _, _, s_default = run(str(tmp_path / "defaults"))
    assert not np.array_equal(_bits(s_default), _bits(want_sc))
