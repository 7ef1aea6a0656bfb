"""Similar items (mmssl_unit_rows + mmssl_recommend_topk through mmssl_b200/similar.py) on the H100: the unit rows against a float64
F.normalize at every width, exact lists on tables whose cosines are exact in fp32, random tables at Baby and Sports shape in all
three spaces against float64 (the modality projections computed from the features and weights in float64), feature queries of
new items, the chunked export, a two-rank row-sharded export read back bitwise the one-GPU lists, and ``Trainer.similar_items``.
The bodies also run on the CPU emulator (tests/test_emu_similar.py)."""
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_zz_recommend import _bits, trainer

pytestmark = pytest.mark.gpu
WIDTHS = (32, 64, 96, 128, 192, 256)
EPS = 1e-12


def unit64(x):
    """float64 F.normalize of the rows of x."""
    x = np.asarray(x, np.float64)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), EPS)


def brute_force(q, c, query_ids, k, exclude_self):
    """float64 lists of the query rows q against the candidate rows c: sorted by (-score, id), the query's own id dropped when
    exclude_self, -1 / 0 past the end."""
    s = q @ c.T
    ids = np.full((q.shape[0], k), -1, np.int64)
    sc = np.zeros((q.shape[0], k))
    for r in range(q.shape[0]):
        keep = np.arange(c.shape[0])
        if exclude_self:
            keep = keep[keep != query_ids[r]]
        order = keep[np.lexsort((keep, -s[r, keep]))][:k]
        ids[r, :order.size] = order
        sc[r, :order.size] = s[r, order]
    return ids, sc


def check_lists(ids, scores, q, c, query_ids, k, exclude_self, extra_tol=0.0, exact=False):
    """Device lists against the float64 brute force of the float64 unit rows q (queries) / c (catalogue).  Per rank the float64
    score of the returned item equals the brute force's within the fp32 band of a d-term dot product of unit rows (plus
    extra_tol: the distance of the device's unit rows from q and c, for tables computed on the device); the set of a list differs
    only by items inside that band of the k-th score; the query itself never appears; padding is -1 / 0; the fp32 scores are
    non-increasing and equal scores keep the lower id first.  exact: every score is exact in fp32, the lists must be equal."""
    ids = ids.cpu().numpy().astype(np.int64) if torch.is_tensor(ids) else np.asarray(ids, np.int64)
    scores = scores.cpu().numpy() if torch.is_tensor(scores) else np.asarray(scores)
    want, want_sc = brute_force(q, c, query_ids, k, exclude_self)
    assert ids.shape == (q.shape[0], k) and scores.shape == (q.shape[0], k)
    if exact:
        assert np.array_equal(ids, want)
        assert np.array_equal(scores.astype(np.float64), want_sc)
        return
    d = q.shape[1]
    s64 = q @ c.T
    mag = np.abs(q) @ np.abs(c).T
    for r in range(q.shape[0]):
        tol = 2.0 * d * 2.0 ** -24 * float(mag[r].max()) + extra_tol + 1e-30
        m = int((want[r] >= 0).sum())
        assert (ids[r, :m] >= 0).all() and (ids[r, m:] == -1).all() and (scores[r, m:] == 0).all(), r
        got = ids[r, :m]
        assert np.unique(got).size == m, r
        if exclude_self:
            assert not (got == query_ids[r]).any(), r
        np.testing.assert_allclose(s64[r, got], want_sc[r, :m], rtol=0, atol=tol)
        np.testing.assert_allclose(scores[r, :m].astype(np.float64), s64[r, got], rtol=0, atol=tol)
        assert (np.diff(scores[r, :m]) <= 0).all(), r
        tie = np.diff(scores[r, :m]) == 0
        assert (np.diff(got)[tie] > 0).all(), r
        extra = np.setdiff1d(got, want[r, :m])
        if extra.size:
            assert m == k and (np.abs(s64[r, extra] - want_sc[r, m - 1]) <= 2 * tol).all(), r


# ------------------------------------------------------------------ 1. unit rows
def run_unit_rows(d, device="cuda", n=37):
    """Ragged leading dimensions in and out, zero rows, rows below 1e-12 and huge rows against float64 F.normalize; columns past
    d of the output untouched; a row's bits the same at every n and at every position in the launch."""
    from mmssl_b200 import ops
    rng = np.random.default_rng(d)
    ldx, ldo = d + 12, d + 4
    xb = rng.standard_normal((n, ldx)).astype(np.float32)
    xb[3] = 0.0
    xb[5, :d] *= np.float32(1e-15)                    # |x| ~ 1e-14: below the eps, x / 1e-12
    xb[6, :d] = 0.0
    xb[6, d - 1] = np.float32(3e-13)
    xb[7, :d] *= np.float32(1e17)
    xb[8, :d] = np.float32(1e-30)                     # |x|^2 underflows
    x = torch.from_numpy(xb).to(device)[:, :d]
    ob = torch.full((n, ldo), 7.0, dtype=torch.float32, device=device)
    out = ops.unit_rows(x, ob[:, :d])
    got = out.cpu().numpy().astype(np.float64)
    want = unit64(xb[:, :d])
    tol = (d + 8) * 2.0 ** -24 * np.abs(want) + 1e-37
    assert (np.abs(got - want) <= tol).all(), float(np.abs(got - want).max())
    assert (ob[:, d:].cpu() == 7.0).all()
    assert (got[3] == 0).all()
    ref = _bits(out)
    for m in (1, 9, n - 1):
        part = ops.unit_rows(x[:m])
        assert np.array_equal(_bits(part), np.ascontiguousarray(out[:m].cpu().numpy()).view(np.uint8)), m
    shifted = ops.unit_rows(x[5:])                    # every row at another lane group and block
    assert np.array_equal(_bits(shifted), np.ascontiguousarray(out[5:].cpu().numpy()).view(np.uint8))
    return ref


@pytest.mark.parametrize("d", WIDTHS)
def test_unit_rows(d):
    run_unit_rows(d, n=3001)


# ------------------------------------------------------------------ 2. exact lists
def exact_table(n, d, seed, zero_rows=()):
    """Rows with entries in {-1, 0, 1} and exactly 4 non-zeros: unit entries are +-0.5, every cosine a multiple of 0.25, exact in
    fp32, with many exact ties (and duplicate rows)."""
    rng = np.random.default_rng(seed)
    t = np.zeros((n, d), np.float32)
    for r in range(n):
        t[r, rng.choice(d, 4, replace=False)] = rng.choice([-1.0, 1.0], 4)
    t[list(zero_rows)] = 0.0
    return t


def run_exact(k, n=150, d=32, device="cuda", seed=1):
    from mmssl_b200.similar import SimilarItems
    t = exact_table(n, d, seed, zero_rows=(2, 77))
    sim = SimilarItems(torch.from_numpy(t).to(device), k)
    items = np.array([0, 2, 77, n - 1, 5, 5, 33] + list(range(40, 60)), np.int64)
    ids, sc = sim.topk(items)
    assert ids.dtype == torch.int64 and sc.dtype == torch.float32
    u = unit64(t)
    check_lists(ids, sc, u[items], u, items, k, True, exact=True)
    got = ids.cpu().numpy()
    assert not (got == items[:, None]).any()
    if k >= n:
        assert ((got >= 0).sum(1) == n - 1).all() and (got[:, n - 1:] == -1).all()
    assert (sc[1].cpu() == 0).all() and (got[1, :min(k, n - 1)] == np.delete(np.arange(n), 2)[:min(k, n - 1)]).all()
    return sim


@pytest.mark.parametrize("k", [1, 64, 65, 200])
def test_exact_lists(k):
    run_exact(k, n=3000 if k < 200 else 150, d=64)


# ------------------------------------------------------------------ 3. random tables, three spaces
def model_problem(I, Dv, Dt, d, seed, device):
    """Engine, parameters and feature stores of a model whose image / text projections are checked against float64."""
    from mmssl_b200.engine import Engine, FeatureStore
    rng = np.random.default_rng(seed)
    fv = rng.standard_normal((I, Dv)).astype(np.float32)
    ft = rng.standard_normal((I, Dt)).astype(np.float32)
    P = {"image_trans.weight": (rng.standard_normal((d, Dv)) / np.sqrt(Dv)).astype(np.float32),
         "image_trans.bias": (0.1 * rng.standard_normal(d)).astype(np.float32),
         "text_trans.weight": (rng.standard_normal((d, Dt)) / np.sqrt(Dt)).astype(np.float32),
         "text_trans.bias": (0.1 * rng.standard_normal(d)).astype(np.float32)}
    Pd = {k: torch.from_numpy(v).to(device) for k, v in P.items()}
    feats = (FeatureStore(torch.from_numpy(fv).to(device)), FeatureStore(torch.from_numpy(ft).to(device)))
    return Engine(d, 2), Pd, feats, P, fv, ft


def proj64(P, fv, ft, space):
    if space == "image":
        return fv.astype(np.float64) @ P["image_trans.weight"].astype(np.float64).T + P["image_trans.bias"]
    return ft.astype(np.float64) @ P["text_trans.weight"].astype(np.float64).T + P["text_trans.bias"]


def _unit_error(sim_unit, u64):
    """Largest row distance of the device's unit rows from float64's (the band it adds to a cosine)."""
    return float(np.linalg.norm(sim_unit.cpu().numpy().astype(np.float64) - u64, axis=1).max())


def run_random(I, d, k, space, n_queries, device="cuda", Dv=96, Dt=40, seed=2):
    from mmssl_b200.similar import SimilarItems
    rng = np.random.default_rng(seed)
    items = np.concatenate([[0, I - 1], rng.choice(I, n_queries, replace=False)]).astype(np.int64)
    if space == "model":
        t = rng.standard_normal((I, d)).astype(np.float32)
        t[7] = 0.0
        sim = SimilarItems(torch.from_numpy(t).to(device), k)
        u = unit64(t)
    else:
        eng, Pd, feats, P, fv, ft = model_problem(I, Dv, Dt, d, seed, device)
        sim = SimilarItems.from_model(eng, Pd, feats, None, k, space)
        u = unit64(proj64(P, fv, ft, space))
    err = _unit_error(sim.unit, u)
    assert err < 1e-4, err               # fp32-class: a bf16 projection would be ~1e-2
    ids, sc = sim.topk(items)
    check_lists(ids, sc, u[items], u, items, k, True, extra_tol=2 * err)
    return sim


@pytest.mark.parametrize("space", ["model", "image", "text"])
@pytest.mark.parametrize("k", [20, 100])
@pytest.mark.parametrize("name", ["baby", "sports"])
def test_random_tables_at_dataset_shape(name, k, space):
    from mmssl_b200.synthetic import CONFIGS
    _, I, _, d, *_ = CONFIGS[name]
    run_random(I, d, k, space, 300, Dv=4096, Dt=384)


# ------------------------------------------------------------------ 4. feature queries
def run_features(I, d, k, space, device="cuda", Dv=96, Dt=40, seed=3):
    """Copies of catalogue items' feature rows as new items: each projects to its item's bits (the K split planned for the
    catalogue), so the item comes first with a score within 1e-6 of 1; the lists match float64 with nothing excluded."""
    from mmssl_b200.similar import SimilarItems
    eng, Pd, feats, P, fv, ft = model_problem(I, Dv, Dt, d, seed, device)
    sim = SimilarItems.from_model(eng, Pd, feats, None, k, space)
    js = np.array([0, I - 1, 5, 5, I // 2, 17], np.int64)
    q, _ = sim._feature_queries(fv[js], ft[js])
    assert np.array_equal(_bits(q), _bits(sim.unit[torch.from_numpy(js).to(sim.unit.device)]))
    ids, sc = sim.topk_features(fv[js], ft[js])
    got, s = ids.cpu().numpy(), sc.cpu().numpy()
    assert (got[:, 0] == js).all() and (np.abs(s[:, 0] - 1.0) <= 1e-6).all()
    u = unit64(proj64(P, fv, ft, space))
    check_lists(ids, sc, u[js], u, js, k, False, extra_tol=2 * _unit_error(sim.unit, u))
    e_ids, e_sc = sim.topk_features(fv[:0], ft[:0])
    assert e_ids.shape == (0, k) and e_sc.shape == (0, k)
    with pytest.raises(ValueError, match="image"):
        SimilarItems(sim.unit, k).topk_features(fv[js], ft[js])
    check_feature_widths(sim, fv[js], ft[js], Dv, Dt)
    return sim


def check_feature_widths(sim, fv, ft, Dv, Dt):
    """Feature rows narrower or wider than the trained widths (image Dv, text Dt) are refused, naming the widths the model takes
    (the tensor-core GEMM would read the first columns of W for narrower rows)."""
    want = f"image {Dv} / text {Dt}"
    pad = lambda a, n: np.concatenate([a, np.zeros((a.shape[0], n), np.float32)], 1)
    for bad_v, bad_t in ((fv[:, :-8], ft), (fv, ft[:, :-4]), (pad(fv, 8), ft), (fv, pad(ft, 4)), (ft, fv)):
        with pytest.raises(ValueError, match=want):
            sim.topk_features(bad_v, bad_t)


@pytest.mark.parametrize("space", ["image", "text"])
def test_feature_queries(space):
    from mmssl_b200.synthetic import CONFIGS
    _, I, _, d, *_ = CONFIGS["baby"]
    run_features(I, d, 20, space, Dv=4096, Dt=384)


# ------------------------------------------------------------------ 5. export
def run_export(tmp_path, k, I=300, d=32, chunk=7, device="cuda"):
    """Chunked export (chunk does not divide n) == one topk call, bitwise; read() returns it; each reader refuses the other's
    directory; no temporary file is left."""
    from mmssl_b200 import recommend, similar
    t = np.random.default_rng(5).standard_normal((I, d)).astype(np.float32)
    sim = similar.SimilarItems(torch.from_numpy(t).to(device), k)
    items = np.concatenate([np.arange(I), [3, 3, 0]]).astype(np.int64)
    ids, sc = sim.topk(items)
    assert items.size % chunk
    out = str(tmp_path / "sim")
    assert sim.export(items, out, chunk=chunk) == items.size
    q, i, s = similar.read(out)
    assert i.dtype == np.int32 and s.dtype == np.float32 and q.dtype == np.int64
    assert np.array_equal(q, items) and np.array_equal(i, ids.cpu().numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(sc))
    assert sorted(os.listdir(out)) == ["ids.npy", "items.npy", "manifest.json", "scores.npy"]
    with pytest.raises(ValueError, match="similar items"):
        recommend.read(out)
    rec_dir = str(tmp_path / "rec")
    recommend.Recommender(torch.from_numpy(t).to(device), similar.empty_csr(4, device), k).export(torch.from_numpy(t[:4]).to(device),
                                                                                                 [0, 1, 2, 3], rec_dir)
    with pytest.raises(ValueError, match="recommendations"):
        similar.read(rec_dir)
    assert recommend.read(rec_dir)[0].tolist() == [0, 1, 2, 3]
    # an export of one kind over the other's: the superseded export's row-id file goes too, nothing of it is left behind
    sim.export([1, 2], rec_dir)
    assert sorted(os.listdir(rec_dir)) == ["ids.npy", "items.npy", "manifest.json", "scores.npy"]
    assert similar.read(rec_dir)[0].tolist() == [1, 2]
    recommend.Recommender(torch.from_numpy(t).to(device), similar.empty_csr(4, device), k).export(torch.from_numpy(t[:4]).to(device),
                                                                                                 [3], rec_dir)
    assert sorted(os.listdir(rec_dir)) == ["ids.npy", "manifest.json", "scores.npy", "users.npy"]
    return sim


@pytest.mark.parametrize("k", [20, 100])
def test_export_equals_topk(tmp_path, k):
    run_export(tmp_path, k, I=5000, d=64, chunk=1000)


# ------------------------------------------------------------------ 6. row-sharded, both ranks in one process
def run_sharded_one_process(tmp_path, I=301, d=32, k=10, device="cuda", Dv=48, Dt=24):
    """Both ranks of a world-2 ShardedSimilarItems in one process (odd I: the last block is padded), the unit-table gather
    replaced by the gathered blocks: in every space the export read back and topk are bitwise the one-GPU SimilarItems's.  The
    modality blocks are projected as RowShardedHotStep.projections does (the split planned for the catalogue): bitwise the
    one-GPU projection."""
    from mmssl_b200 import ops, similar
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.parallel import RowPartition
    pi = RowPartition(I, 2)
    assert I % 2 and pi.block * 2 > I
    rng = np.random.default_rng(8)
    eng, Pd, feats, P, fv, ft = model_problem(I, Dv, Dt, d, 8, device)
    items = np.concatenate([rng.permutation(I), [0, I - 1, 0]]).astype(np.int64)
    tables = {"model": torch.from_numpy(rng.standard_normal((I, d)).astype(np.float32)).to(device)}
    blocks = {"model": [pi.local(tables["model"], r) for r in range(2)]}
    full = similar.project(eng, Pd, feats)
    for j, space in enumerate(("image", "text")):
        tables[space] = full[j]
        blocks[space] = []
        for r in range(2):
            fs = tuple(FeatureStore(pi.local(f.fp32, r).contiguous()) for f in feats)
            blk = similar.project(eng, Pd, fs, plan_rows=I)[j]
            lo, hi = pi.bounds(r)
            assert np.array_equal(_bits(blk[:hi - lo]), _bits(full[j][lo:hi].contiguous())), (space, r)
            blocks[space].append(blk)
    for space in similar.SPACES:
        one = similar.SimilarItems(tables[space], k, space)
        for name, its in (("all", items), ("rank1_only", np.arange(pi.block, I)[::-1].copy())):
            out = str(tmp_path / f"{space}_{name}")
            one.export(its[:5], out)
            units = [ops.unit_rows(b) for b in blocks[space]]
            gathered = torch.cat(units)[:I]
            for r in range(2):
                sh = similar.ShardedSimilarItems(pi, r, k, space, device=device)
                sh.gather = lambda unit_local: gathered
                sh.export_id = lambda: 12345
                got_i, got_s, pos = sh.topk(blocks[space][r], its)
                wi, ws = one.topk(its[pos])
                assert torch.equal(got_i, wi) and np.array_equal(_bits(got_s), _bits(ws)), (space, name, r)
                sh.export(blocks[space][r], its, out, chunk=4)
            q, i, s = similar.read(out)
            want_q = np.sort(its, kind="stable")
            wi, ws = one.topk(want_q)
            assert np.array_equal(q, want_q) and np.array_equal(i, wi.cpu().numpy().astype(np.int32)), (space, name)
            assert np.array_equal(_bits(s), _bits(ws)), (space, name)
            assert not os.path.exists(os.path.join(out, "manifest.json"))


def test_sharded_world_two(tmp_path):
    run_sharded_one_process(tmp_path, I=7051, d=64, k=20, Dv=4096, Dt=384)


# ------------------------------------------------------------------ 7. Trainer
def run_trainer(tmp_path, device="cuda", k=10):
    """Two epochs, then similar_items in every space == SimilarItems on the tables of the eval-mode forward (the lists within the
    float64 band), and a fresh Trainer that loads the checkpoint gives the same lists bitwise; feature queries of copies of
    catalogue rows put their item first."""
    from mmssl_b200 import similar
    path = str(tmp_path / "run.ckpt")
    tr = trainer(device, ckpt=path)
    tr.train()
    items = np.arange(tr.n_items, dtype=np.int64)[::-1].copy()
    hs = tr.step.hs
    outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, None, want_sumsq=False)
    xv, xt = similar.project(hs.engine, hs.P, hs.feats)
    got = {}
    for space, t in (("model", outs[1]), ("image", xv), ("text", xt)):
        ids, sc = tr.similar_items(items, k, space)
        u = ops_unit(t)
        check_lists(ids, sc, u[items], u, items, k, True, extra_tol=2 * _unit_error(similar.ops.unit_rows(t), u))
        got[space] = (ids, sc)
    fresh = trainer(device, epochs=2)
    fresh.load(path)
    for space, (i0, s0) in got.items():
        i1, s1 = fresh.similar_items(items, k, space)
        assert np.array_equal(i1.cpu().numpy(), i0.cpu().numpy()) and np.array_equal(_bits(s1), _bits(s0)), space
    img, txt = np.asarray(tr.data.image_feats), np.asarray(tr.data.text_feats)
    js = np.array([0, 3, tr.n_items - 1])
    feats = {"image": img, "text": txt}
    for space in ("image", "text"):
        ids, sc = tr.similar_to_features(img[js], txt[js], k, space)
        first = ids[:, 0].cpu().numpy()                 # the item itself, or an item with the same features and a lower id
        assert (first <= js).all() and np.array_equal(feats[space][first], feats[space][js]), space
        assert (np.abs(sc[:, 0].cpu().numpy() - 1) <= 1e-6).all(), space
    with pytest.raises(ValueError):
        tr.similar_items(items, k, "audio")
    with pytest.raises(ValueError, match="outside"):
        tr.similar_items([tr.n_items], k)
    return tr


def ops_unit(t):
    """float64 unit rows of a device table."""
    return unit64(t.detach().cpu().numpy())


def test_trainer_similar_items(tmp_path):
    run_trainer(tmp_path)
