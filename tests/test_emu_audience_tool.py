"""tools/recommend.py --audience end to end on the CPU emulator: a Trainer run on tests/golden/dataset_small saves its checkpoint,
the tool rebuilds the Trainer from it and exports the audiences of every item, or of the items of an --items file; the files read
back with ``audience.read`` equal ``Trainer.audience`` of the saved run, for both exclusion sets, and --items without --audience
is refused.  (The row-sharded mode runs in tests/test_dist_emu_audience.py.)"""
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
def test_audience_tool_on_a_trainer_checkpoint(monkeypatch, tmp_path, capsys, exclude):
    from mmssl_b200 import audience, recommend
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    from mmssl_b200.dataset import ReferenceDataset
    real = ReferenceDataset.load.__func__
    monkeypatch.setattr(ReferenceDataset, "load", classmethod(lambda cls, path, mmap_features=True: real(cls, path, False)))
    ckpt = str(tmp_path / "run.ckpt")
    tr = trainer("cpu", epochs=1, ckpt=ckpt)
    tr.train()
    listed = np.array([7, 0, 7, tr.n_items - 1], np.int64)
    np.save(str(tmp_path / "items.npy"), listed)

    def run(out, *extra):
        monkeypatch.setattr(sys, "argv", ["recommend.py", os.path.join(GOLD, "dataset_small"), "--checkpoint", ckpt, "--k", "6",
                                          "--exclude", exclude, "--out", out, "--chunk", "5", *extra])
        runpy.run_path(os.path.join(ROOT, "tools", "recommend.py"), run_name="__main__")
        return capsys.readouterr().out

    for name, items, extra in (("all", np.arange(tr.n_items), []), ("listed", listed, ["--items", str(tmp_path / "items.npy")])):
        out = str(tmp_path / name)
        assert '"audiences": %d' % items.size in run(out, "--audience", *extra)
        assert sorted(os.listdir(out)) == ["ids.npy", "items.npy", "manifest.json", "scores.npy"]
        q, i, s = audience.read(out)
        want_ids, want_sc = tr.audience(items, 6, exclude)
        assert np.array_equal(q, items) and np.array_equal(i, want_ids.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(want_sc))
        with pytest.raises(ValueError, match="audience"):
            recommend.read(out)
    with pytest.raises(SystemExit):
        run(str(tmp_path / "bad"), "--items", str(tmp_path / "items.npy"))
