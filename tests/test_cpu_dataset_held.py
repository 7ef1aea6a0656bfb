"""Held-out sets in the shard format: ``write_shards`` writes ``val`` / ``test`` as CSR over users, ``ShardedDataset.held`` and
``train_rows`` give every rank the rows of its user block, and together the ranks' blocks are ``ReferenceDataset``'s
``val_set`` / ``test_set`` / ``train_items``.  A directory written before the held-out files existed still opens and trains
(bitwise the same step), and ``held`` says which files it misses."""
import json
import os

import numpy as np
import pytest
import torch

from mmssl_b200.dataset import HELD, ReferenceDataset, ShardedDataset, held_csr, write_shards
from mmssl_b200.parallel import RowPartition

ROOT = os.path.join(os.path.dirname(__file__), "golden", "dataset_small")


def _train_mat_rows(ds):
    """user -> sorted items of train_mat: the training rows a shard directory holds."""
    R = ds.train_mat.tocsr()
    R.sort_indices()
    return {u: R.indices[R.indptr[u]:R.indptr[u + 1]].tolist() for u in range(R.shape[0]) if R.indptr[u + 1] > R.indptr[u]}


def _reassemble(blocks):
    out = {}
    for blk in blocks:
        for r in range(blk.hi - blk.lo):
            row = blk.indices[blk.indptr[r]:blk.indptr[r + 1]]
            if row.size:
                out[blk.lo + r] = row.tolist()
    return out


@pytest.mark.parametrize("world", [1, 2, 3])
def test_held_and_train_rows_reassemble_reference_sets(tmp_path, world):
    ds = ReferenceDataset.load(ROOT)
    meta = write_shards(ds, str(tmp_path))
    assert meta["format"] == "mmssl_b200.shards.v1" and set(meta["held"]) == set(HELD)
    assert meta["held"]["test"]["nnz"] == sum(len(v) for v in ds.test_set.values())
    got = {"val": [], "test": [], "train": []}
    for rank in range(world):
        sh = ShardedDataset.open(str(tmp_path), rank, world)
        part = RowPartition(ds.train_mat.shape[0], world)
        for name, blk in (("val", sh.held("val")), ("test", sh.held("test")), ("train", sh.train_rows())):
            assert blk.indptr.dtype == np.int64 and blk.indices.dtype == np.int32 and blk.values is None
            assert blk.indptr.shape == (part.block + 1,) and blk.indptr[0] == 0
            assert (blk.lo, blk.hi) == part.bounds(rank) and blk.shape == (part.block, sh.n_items)
            assert np.all(blk.indptr[blk.hi - blk.lo:] == blk.indptr[-1])          # padding rows are empty
            assert blk.to_scipy().nnz == blk.indices.size
            got[name].append(blk)
    sort = lambda d: {u: sorted(v) for u, v in d.items()}
    assert _reassemble(got["val"]) == sort(ds.val_set)
    assert _reassemble(got["test"]) == sort(ds.test_set)
    # the training rows are the pattern of train_mat (the graph the model trains on); dataset_small's train.json lists user 5
    # with no items (the loader drops it) while train_mat holds its row, so that one row is train_mat's alone
    train = _reassemble(got["train"])
    assert train == _train_mat_rows(ds)
    assert {u: v for u, v in train.items() if u in ds.train_items} == sort(ds.train_items)
    assert set(train) - set(ds.train_items) == {5}
    with pytest.raises(ValueError):
        ShardedDataset.open(str(tmp_path), 0, world).held("train")


def test_held_csr_keeps_duplicates_sorted():
    ip, ix = held_csr({3: [5, 1, 5], 0: [2], 1: []}, 5)
    assert ip.tolist() == [0, 1, 1, 1, 4, 4] and ix.tolist() == [2, 1, 5, 5]
    with pytest.raises(ValueError):
        held_csr({5: [1]}, 5)


def _old_directory(tmp_path):
    """A shard directory as written before the held-out sets were part of the format."""
    ds = ReferenceDataset.load(ROOT)
    new, old = tmp_path / "new", tmp_path / "old"
    write_shards(ds, str(new))
    write_shards(ds, str(old))
    for split in HELD:
        for suffix in ("indptr.i64", "indices.i32"):
            os.remove(old / f"{split}.{suffix}")
    meta = json.loads((old / "meta.json").read_text())
    del meta["held"]
    (old / "meta.json").write_text(json.dumps(meta))
    return ds, str(new), str(old)


def test_directory_without_held_files_opens_trains_and_names_them(tmp_path, monkeypatch):
    ds, new, old = _old_directory(tmp_path)
    sh = ShardedDataset.open(old, 0, 1)
    with pytest.raises(ValueError, match=r"val\.indptr\.i64 / val\.indices\.i32 are missing"):
        sh.held("val")
    with pytest.raises(ValueError, match=r"test\.indptr\.i64"):
        sh.held("test")
    assert sh.train_rows().indices.size == sh.meta["operands"]["ui"]["nnz"]
    assert sh.bytes_touched() == ShardedDataset.open(new, 0, 1).bytes_touched()
    # one row-sharded step (world 1, the real kernels under the emulator) from either directory: bitwise the same
    from tests.cuemu import harness
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    from mmssl_b200.engine import LIVE
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
    U, I = ds.train_mat.shape
    d, B = 64, 8
    g = torch.Generator().manual_seed(4)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, ds.image_feats.shape[1]), "image_trans.bias": torch.zeros(d),
         "text_trans.weight": xav(d, ds.text_feats.shape[1]), "text_trans.bias": torch.zeros(d),
         "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    users = torch.randperm(U, generator=g)[:B]
    pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
    cfg = HotStepConfig(embed_size=d, n_layers=2, batch_size=B, drop_rate=0.0, proj_impl="simt")
    runs = []
    for root in (new, old):
        Pl, fl, gl, pu, pi = shard_problem_from_disk(root, P, 0, 1, "cpu")
        st = RowShardedHotStep(Pl, fl, gl, cfg, B, pu, pi, 0)
        st.set_indices(users, pos, neg)
        runs.append((st.run().clone(), {k: st.P[k].clone() for k in LIVE}))
    (o_new, p_new), (o_old, p_old) = runs
    assert torch.equal(o_new, o_old)
    assert all(torch.equal(p_new[k], p_old[k]) for k in LIVE)


@pytest.mark.parametrize("flag", ["part", "full"])
def test_sharded_evaluator_from_shards_world_one(tmp_path, monkeypatch, flag):
    """World 1 (no process group): ShardedEvaluator.from_shards on the shard arrays == Evaluator on the reference's dicts."""
    from tests.cuemu import harness
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    from mmssl_b200.evaluate import Evaluator, ShardedEvaluator
    ds = ReferenceDataset.load(ROOT)
    write_shards(ds, str(tmp_path))
    sh = ShardedDataset.open(str(tmp_path), 0, 1)
    U, I = sh.n_users, sh.n_items
    rng = np.random.default_rng(3)
    ua = torch.from_numpy(rng.integers(-2, 3, (U, 16)).astype(np.float32))
    ia = torch.from_numpy(rng.integers(-2, 3, (I, 16)).astype(np.float32))
    ev = Evaluator(_train_mat_rows(ds), ds.test_set, ds.val_set, U, I, [2, 5, 10], device="cpu", test_flag=flag)
    se = ShardedEvaluator.from_shards(sh, [2, 5, 10], flag, device="cpu")
    for is_val, rows in ((False, ds.test_set), (True, ds.val_set)):
        users = sorted(rows)[::-1]
        want, got = ev.rank(ua, ia, users, is_val), se.rank(ua, ia, users, is_val)
        for k in ("result", "per_user", "ranked", "ranked_scores", "hits") + (("auc",) if flag == "full" else ()):
            assert np.array_equal(want[k].numpy().view(np.uint8), got[k].numpy().view(np.uint8)), k
        assert got["positions"].tolist() == list(range(len(users)))
