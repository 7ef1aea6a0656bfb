"""tools/similar_items.py end to end on the CPU emulator: a Trainer run on tests/golden/dataset_small saves its checkpoint, the tool
rebuilds the Trainer from the checkpoint and the dataset directory and exports every item's list, in each space, and the lists of
new items given by feature files; the files read back with ``similar.read`` are bitwise ``Trainer.similar_items`` /
``Trainer.similar_to_features`` of the saved run."""
import os
import runpy
import sys

import numpy as np
import pytest
import torch

from tests.cuemu import harness
from tests.test_gpu_zz_recommend import GOLD, _bits, trainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def trained(monkeypatch, tmp_path):
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
    return tr, ckpt


def _run(monkeypatch, capsys, ckpt, out, *extra):
    from mmssl_b200 import similar
    monkeypatch.setattr(sys, "argv", ["similar_items.py", os.path.join(GOLD, "dataset_small"), "--checkpoint", ckpt, "--k", "7",
                                      "--out", out, "--chunk", "5", "--id-cat-rate", "0.2", "--model-cat-rate", "0.7", *extra])
    runpy.run_path(os.path.join(ROOT, "tools", "similar_items.py"), run_name="__main__")
    assert '"queries": ' in capsys.readouterr().out
    return similar.read(out)


@pytest.mark.parametrize("space", ["model", "image", "text"])
def test_similar_tool_on_a_trainer_checkpoint(trained, monkeypatch, tmp_path, capsys, space):
    tr, ckpt = trained
    want_ids, want_sc = tr.similar_items(np.arange(tr.n_items), 7, space)
    out = str(tmp_path / f"out_{space}")
    q, i, s = _run(monkeypatch, capsys, ckpt, out, "--space", space)
    assert sorted(os.listdir(out)) == ["ids.npy", "items.npy", "manifest.json", "scores.npy"]
    assert np.array_equal(q, np.arange(tr.n_items))
    assert np.array_equal(i, want_ids.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(want_sc))


def test_similar_tool_feature_queries(trained, monkeypatch, tmp_path, capsys):
    tr, ckpt = trained
    img, txt = np.asarray(tr.data.image_feats)[[4, 0, 9]], np.asarray(tr.data.text_feats)[[4, 0, 9]]
    np.save(str(tmp_path / "img.npy"), img)
    np.save(str(tmp_path / "txt.npy"), txt)
    want_ids, want_sc = tr.similar_to_features(img, txt, 7, "text")
    q, i, s = _run(monkeypatch, capsys, ckpt, str(tmp_path / "feat"), "--space", "text", "--features", str(tmp_path / "img.npy"),
                   str(tmp_path / "txt.npy"))
    assert q.tolist() == [0, 1, 2]
    assert np.array_equal(i, want_ids.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(want_sc))
    with pytest.raises(SystemExit):
        _run(monkeypatch, capsys, ckpt, str(tmp_path / "bad"), "--features", str(tmp_path / "img.npy"), str(tmp_path / "txt.npy"))
    np.save(str(tmp_path / "img_narrow.npy"), img[:, :-2])           # a feature file of another width than the trained one
    with pytest.raises(ValueError, match="image %d / text %d" % (img.shape[1], txt.shape[1])):
        _run(monkeypatch, capsys, ckpt, str(tmp_path / "narrow"), "--space", "text", "--features", str(tmp_path / "img_narrow.npy"),
             str(tmp_path / "txt.npy"))
    assert not os.path.exists(str(tmp_path / "narrow"))
