"""Recommendations (mmssl_recommend_topk through mmssl_b200/recommend.py) on the H100: the lists against a float64 brute force
(exact wherever neighbouring ranks are further apart than fp32 rounding, the same set across a near-tie), bitwise
``Evaluator.rank``'s ranked / ranked_scores with Ks = [k] at Baby and Sports shape for k = 20 and 100, the chunked export
bitwise one ``topk`` call, a two-rank row-sharded export read back bitwise the one-GPU lists, and ``Trainer.recommend``.  The
bodies also run on the CPU emulator (tests/test_emu_recommend.py)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _csr(rows, U):
    indptr = np.zeros(U + 1, np.int64)
    for u, its in rows.items():
        indptr[u + 1] = len(set(its))
    np.cumsum(indptr, out=indptr)
    indices = np.concatenate([np.zeros(0, np.int64)] + [np.sort(np.unique(np.asarray(rows[u], np.int64))) for u in range(U) if u in rows])
    return indptr, indices


def _bits(t):
    return np.ascontiguousarray(t.cpu().numpy() if torch.is_tensor(t) else t).view(np.uint8)


def brute_force(ua, ia, users, excl, k):
    """float64 lists: excluded items dropped, sorted by (-score, id), -1 past the end.  Returns (ids [n, k], scores64 [n, k])."""
    indptr, indices = excl
    s = ua.astype(np.float64) @ ia.astype(np.float64).T
    ids = np.full((len(users), k), -1, np.int64)
    sc = np.zeros((len(users), k))
    for r, u in enumerate(users):
        keep = np.setdiff1d(np.arange(ia.shape[0]), indices[indptr[u]:indptr[u + 1]])
        order = keep[np.lexsort((keep, -s[u, keep]))][:k]
        ids[r, :order.size] = order
        sc[r, :order.size] = s[u, order]
    return ids, sc


def check_lists(ids, scores, ua, ia, users, excl, k, exact=False):
    """ids [n, k] / scores [n, k] of the device against the brute force.  Per rank, the float64 score of the returned item equals
    the brute force's within the fp32 rounding of a d-term dot product (so the lists agree except across near-ties); the set of a
    list differs only by items inside that band of the k-th score; excluded items never appear, padding is -1 / 0; the fp32 scores
    are the returned items' within the same band, non-increasing, and equal scores keep the lower id first.  exact: the embeddings
    make every score exact in fp32, so the lists must be the brute force's."""
    ids = ids.cpu().numpy().astype(np.int64) if torch.is_tensor(ids) else ids
    scores = scores.cpu().numpy() if torch.is_tensor(scores) else scores
    want, want_sc = brute_force(ua, ia, users, excl, k)
    assert ids.shape == (len(users), k) and scores.shape == (len(users), k)
    if exact:
        assert np.array_equal(ids, want)
    d = ua.shape[1]
    mag = np.abs(ua.astype(np.float64)) @ np.abs(ia.astype(np.float64)).T
    indptr, indices = excl
    s64 = ua.astype(np.float64) @ ia.astype(np.float64).T
    for r, u in enumerate(users):
        tol = 2.0 * d * 2.0 ** -24 * float(mag[u].max()) + 1e-30
        m = int((want[r] >= 0).sum())
        assert (ids[r, :m] >= 0).all() and (ids[r, m:] == -1).all() and (scores[r, m:] == 0).all(), r
        got = ids[r, :m]
        assert np.unique(got).size == m and not np.isin(got, indices[indptr[u]:indptr[u + 1]]).any(), r
        np.testing.assert_allclose(s64[u, got], want_sc[r, :m], rtol=0, atol=tol)
        np.testing.assert_allclose(scores[r, :m].astype(np.float64), s64[u, got], rtol=0, atol=tol)
        assert (np.diff(scores[r, :m]) <= 0).all(), r
        tie = np.diff(scores[r, :m]) == 0
        assert (np.diff(got)[tie] > 0).all(), r
        extra = np.setdiff1d(got, want[r, :m])
        if extra.size:
            assert m == k and (np.abs(s64[u, extra] - want_sc[r, m - 1]) <= 2 * tol).all(), r


def problem(U, I, d, seed, kind="normal", n_excl=(0, 60)):
    rng = np.random.default_rng(seed)
    if kind == "ties":            # small integers: exact scores, many equal; repeated item rows tie exactly
        ua = rng.integers(-2, 3, (U, d)).astype(np.float32)
        ia = rng.integers(-2, 3, (I, d)).astype(np.float32)
        ia[I // 2:I // 2 + 20] = ia[3]
    else:
        ua = rng.standard_normal((U, d)).astype(np.float32)
        ia = rng.standard_normal((I, d)).astype(np.float32)
    train = {u: rng.choice(I, size=min(int(rng.integers(*n_excl)), I), replace=False).tolist() for u in range(U)}
    train = {u: v for u, v in train.items() if v}
    return ua, ia, train


def run_lists(k, U=13, I=300, d=8, kind="normal", seed=1, device="cuda"):
    """One user with every item excluded, one with none, repeated users, n_items not a multiple of 128."""
    from mmssl_b200.recommend import Recommender
    ua, ia, train = problem(U, I, d, seed, kind)
    train[2] = list(range(I))
    train.pop(5, None)
    users = np.array([4, 0, 2, 5, 9, 1, 3, 6, 7, 8, 10, 11, 12, 4, 5], np.int64)
    rec = Recommender.from_rows(torch.from_numpy(ia).to(device), train, {}, {}, U, k)
    ids, sc = rec.topk(torch.from_numpy(ua).to(device), users)
    assert ids.dtype == torch.int64 and sc.dtype == torch.float32
    check_lists(ids, sc, ua, ia, users, _csr(train, U), k, exact=kind == "ties")
    assert (ids[2] == -1).all()
    return ids, sc


@pytest.mark.parametrize("k", [1, 20, 64, 65, 300])
def test_lists_against_brute_force(k):
    run_lists(k, U=40, I=2000, d=64)


def run_against_evaluator(U, I, d, k, n_users, seed=3, device="cuda", train=None, ua=None, ia=None):
    """Recommender.topk with the training rows excluded == Evaluator.rank's ranked / ranked_scores with Ks = [k], bit for bit."""
    from mmssl_b200.evaluate import Evaluator
    from mmssl_b200.recommend import Recommender
    rng = np.random.default_rng(seed)
    if train is None:
        ua, ia, train = problem(U, I, d, seed, n_excl=(0, 40))
    users = rng.permutation(U)[:n_users].astype(np.int64)
    uc, ic = torch.from_numpy(ua).to(device), torch.from_numpy(ia).to(device)
    ev = Evaluator(train, {}, {}, U, I, [k], device=device)
    out = ev.rank(uc, ic, users, False)
    ids, sc = Recommender.from_rows(ic, train, {}, {}, U, k).topk(uc, users)
    assert np.array_equal(ids.cpu().numpy(), out["ranked"].cpu().numpy().astype(np.int64))
    assert np.array_equal(_bits(sc), _bits(out["ranked_scores"]))
    return ids, sc


def _config(name):
    from mmssl_b200.synthetic import CONFIGS, make_bipartite
    U, I, nnz, d, *_ = CONFIGS[name]
    tr = make_bipartite(U, I, nnz, seed=3).tocsr()
    tr.sort_indices()
    rng = np.random.default_rng(2)
    ua = rng.standard_normal((U, d)).astype(np.float32)
    ia = rng.standard_normal((I, d)).astype(np.float32)
    train = {u: tr.indices[tr.indptr[u]:tr.indptr[u + 1]].tolist() for u in range(U) if tr.indptr[u + 1] > tr.indptr[u]}
    return U, I, d, ua, ia, train


@pytest.mark.parametrize("k", [20, 100])
@pytest.mark.parametrize("name", ["baby", "sports"])
def test_bitwise_evaluator_at_dataset_shape(name, k):
    U, I, d, ua, ia, train = _config(name)
    run_against_evaluator(U, I, d, k, U, train=train, ua=ua, ia=ia)


def run_export(tmp_path, k, U=37, I=500, d=16, chunk=7, device="cuda"):
    """Chunked export (chunk does not divide n) == one topk call, bitwise; read() returns it; no temporary file is left."""
    from mmssl_b200 import recommend
    ua, ia, train = problem(U, I, d, 5)
    users = np.concatenate([np.arange(U), [3, 3, 0]]).astype(np.int64)
    uc, ic = torch.from_numpy(ua).to(device), torch.from_numpy(ia).to(device)
    rec = recommend.Recommender.from_rows(ic, train, {}, {}, U, k)
    ids, sc = rec.topk(uc, users)
    assert users.size % chunk
    out = str(tmp_path / "rec")
    assert rec.export(uc, users, out, chunk=chunk) == users.size
    u, i, s = recommend.read(out)
    assert i.dtype == np.int32 and s.dtype == np.float32 and u.dtype == np.int64
    assert np.array_equal(u, users) and np.array_equal(i, ids.cpu().numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(sc))
    assert sorted(os.listdir(out)) == ["ids.npy", "manifest.json", "scores.npy", "users.npy"]
    return rec, uc


@pytest.mark.parametrize("k", [20, 100])
def test_export_equals_topk(tmp_path, k):
    run_export(tmp_path, k, U=3000, I=5000, d=64, chunk=1000)


def run_sharded_one_process(tmp_path, exclude, U=29, I=300, d=16, device="cuda"):
    """Both ranks of a world-2 ShardedRecommender in one process, the item gather replaced by the full table: every rank's export
    read back == the one-GPU Recommender.  Users of rank 1's block only: rank 0 writes empty files.  A one-GPU export in the same
    directory before is superseded; a later export that only rank 0 finished is refused by read(), not mixed with rank 1's files."""
    from mmssl_b200 import recommend
    from mmssl_b200.parallel import RowPartition
    ua, ia, train = problem(U, I, d, 8)
    rng = np.random.default_rng(8)
    test = {u: rng.choice(I, size=3, replace=False).tolist() for u in range(U)}
    val = {u: rng.choice(I, size=2, replace=False).tolist() for u in range(0, U, 2)}
    pu, pi = RowPartition(U, 2), RowPartition(I, 2)
    uc, ic = torch.from_numpy(ua).to(device), torch.from_numpy(ia).to(device)
    one = recommend.Recommender.from_rows(ic, train, test, val, U, 10, exclude)
    for name, users in (("all", rng.permutation(U)), ("one_block", np.arange(pu.block, U)[::-1])):
        out = str(tmp_path / f"{exclude}_{name}")
        one.export(uc, users[:5], out)
        ranks = []
        for r in range(2):
            sh = recommend.ShardedRecommender.from_rows(train, test, val, U, I, pu, pi, r, 10, exclude, device=device)
            sh.gather_items = lambda i_local: ic
            sh.export_id = lambda: 12345
            sh.export(pu.local(uc, r), pi.local(ic, r), users, out, chunk=4)
            ranks.append(sh)
        u, i, s = recommend.read(out)
        want_u = np.sort(users)
        wi, ws = one.topk(uc, want_u)
        assert np.array_equal(u, want_u) and np.array_equal(i, wi.cpu().numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))
        assert not os.path.exists(os.path.join(out, "manifest.json"))
        ranks[0].export_id = lambda: 777                           # a new export that rank 1 never wrote
        ranks[0].export(pu.local(uc, 0), pi.local(ic, 0), users[::2], out, chunk=4)
        with pytest.raises(ValueError, match="different exports"):
            recommend.read(out)


@pytest.mark.parametrize("exclude", ["train", "seen"])
def test_sharded_export_world_two(tmp_path, exclude):
    run_sharded_one_process(tmp_path, exclude, U=2001, I=3000, d=64)


def trainer(device, epochs=2, ckpt="", **over):
    from mmssl_b200.dataset import ReferenceDataset
    from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed
    ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
    ds.image_feats, ds.text_feats = np.array(ds.image_feats), np.array(ds.text_feats)
    args = TrainerArgs(dataset="dataset_small", epoch=epochs, batch_size=16, verbose=1, early_stopping_patience=5, m_topk_rate=0.05,
                       Ks="[2, 5, 10]", seed=5, checkpoint=ckpt, **over)
    set_seed(5)
    return Trainer(ds, args, device=device, log=None)


def run_trainer(tmp_path, device="cuda", k=10):
    """Two epochs, then recommend(users, k, "train") == Evaluator.rank on the tables Trainer.test ranks; a fresh Trainer that
    loads the run's checkpoint recommends the same lists, for both exclusion sets."""
    from mmssl_b200.evaluate import Evaluator
    path = str(tmp_path / "run.ckpt")
    tr = trainer(device, ckpt=path)
    tr.train()
    users = np.arange(tr.n_users, dtype=np.int64)[::-1].copy()
    ids, sc = tr.recommend(users, k, "train")
    hs = tr.step.hs
    outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, None, want_sumsq=False)
    ev = Evaluator(tr.data.train_items, tr.data.test_set, tr.data.val_set, tr.n_users, tr.n_items, [k], device=device)
    want = ev.rank(outs[0], outs[1], users, False)
    assert np.array_equal(ids.cpu().numpy(), want["ranked"].cpu().numpy().astype(np.int64))
    assert np.array_equal(_bits(sc), _bits(want["ranked_scores"]))
    seen = tr.recommend(users, k, "seen")
    fresh = trainer(device, epochs=2)
    fresh.load(path)
    for ex, (i0, s0) in (("train", (ids, sc)), ("seen", seen)):
        i1, s1 = fresh.recommend(users, k, ex)
        assert np.array_equal(i1.cpu().numpy(), i0.cpu().numpy()) and np.array_equal(_bits(s1), _bits(s0)), ex
    with pytest.raises(ValueError):
        tr.recommend(users, k, "everything")
    return tr


def test_trainer_recommend(tmp_path):
    run_trainer(tmp_path)
