"""Audiences (mmssl_b200/audience.py) and the sliced sweep + merge under them (mmssl_recommend_topk_sliced, mmssl_topk_merge) on the
H100.  Every comparison is bitwise: the keys (score bits, then id) are unique, so a list has one right answer.
  * exact model: the audience of item i is the top-k of column i of ``Evaluator.rank``'s own score matrix by the sweep key, the
    item's excluded users dropped -- both buffer routes, every width, exact ties, short lists, an item every user has, empty,
    repeated and unsorted item lists, out-of-range ids;
  * sliced == unsliced for S in {1, 2, 3, 7, > n_cand}, with slice bounds inside a run of tied scores and inside exclusion rows;
  * the merge against a host model of the key, -0.0 / +0.0 scores included, and independent of the lists' order;
  * ``Recommender`` and ``SimilarItems`` forced to slice still give the evaluator's / the unsliced lists;
  * the row-sharded audience at world 2 in one process (the exchange stood in), and ``Trainer.audience``.
The bodies also run on the CPU emulator (tests/test_emu_audience.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_gpu_zz_recommend import _bits, _config, problem

pytestmark = pytest.mark.gpu


def host_key(scores: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """The sweep's key as uint64: order-preserving transform of the fp32 bits, then 0xFFFFFFFF - id (lower id = larger key)."""
    b = np.ascontiguousarray(scores, np.float32).view(np.uint32).astype(np.uint64)
    b = np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000).astype(np.uint64)
    return (b << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - ids.astype(np.uint64))


def host_topk(col: np.ndarray, excluded, k: int):
    """(ids, scores) of the best k entries of one fp32 score column by the key, excluded ids dropped, -1 / 0 past the end."""
    cand = np.setdiff1d(np.arange(col.size), np.asarray(list(excluded), np.int64))
    order = cand[np.argsort(host_key(col[cand], cand))[::-1]][:k]
    ids = np.full(k, -1, np.int64)
    sc = np.zeros(k, np.float32)
    ids[:order.size] = order
    sc[:order.size] = col[order]
    return ids, sc


def exact_model(ua, ia, train, items, k, device):
    """Audience lists of `items` from the evaluator's [users, items] score matrix (the sweep's own scores), transposed."""
    from mmssl_b200.evaluate import Evaluator
    U, I = ua.shape[0], ia.shape[0]
    ev = Evaluator({}, {}, {}, U, I, [1], device=device)
    S = ev.rank(torch.from_numpy(ua).to(device), torch.from_numpy(ia).to(device), np.arange(U), False, want_scores=True)["scores"]
    S = S.cpu().numpy()
    holders = {i: set() for i in range(I)}
    for u, its in train.items():
        for i in its:
            holders[int(i)].add(int(u))
    want = [host_topk(S[:, i], holders[int(i)], k) for i in items]
    return np.array([w[0] for w in want]).reshape(len(items), k), np.array([w[1] for w in want], np.float32).reshape(len(items), k)


def run_exact(k, U=70, I=40, d=8, kind="normal", seed=1, items=None, device="cuda"):
    """Audience.topk == the exact model, bitwise.  Item 0 is held by every user (an empty list), item 1 by none."""
    from mmssl_b200.audience import Audience
    ua, ia, train = problem(U, I, d, seed, kind, n_excl=(0, I // 3))
    if kind == "ties":                                     # 20 copies of one user row: exactly equal scores, lower user first
        ua[U // 2:U // 2 + 20] = ua[3]
    for u in range(U):
        train[u] = sorted((set(train.get(u, [])) | {0}) - {1})
    items = np.array([0, 1, 5, 3, 3, I - 1, 2], np.int64) if items is None else items
    aud = Audience.from_rows(torch.from_numpy(ua).to(device), train, {}, {}, I, k)
    ids, sc = aud.topk(torch.from_numpy(ia).to(device), items)
    want_ids, want_sc = exact_model(ua, ia, train, items, k, device)
    assert ids.dtype == torch.int64 and sc.dtype == torch.float32 and ids.shape == (items.size, k)
    assert np.array_equal(ids.cpu().numpy(), want_ids)
    assert np.array_equal(_bits(sc), _bits(want_sc))
    assert (ids.cpu()[torch.from_numpy(items == 0)] == -1).all() and (ids.cpu()[torch.from_numpy(items == 1)] >= 0).any()
    return aud, ua, ia


@pytest.mark.parametrize("k", [1, 64, 65, 300])
def test_exact_model_both_routes(k):
    run_exact(k, U=600, I=50, d=32)


@pytest.mark.parametrize("d", [32, 64, 96, 128, 192, 256])
def test_exact_model_every_width(d):
    run_exact(20 if d % 64 else 70, U=300, I=30, d=d, seed=d)


def run_queries(device="cuda"):
    """Ties (duplicated user rows), k above the eligible users, empty / repeated / unsorted item lists, out-of-range ids."""
    from mmssl_b200.audience import Audience
    aud, ua, ia = run_exact(9, U=90, I=20, d=8, kind="ties", seed=3, device=device)
    ic = torch.from_numpy(ia).to(device)
    ids, sc = aud.topk(ic, np.zeros(0, np.int64))
    assert ids.shape == (0, 9) and sc.shape == (0, 9)
    run_exact(200, U=90, I=20, d=8, seed=6, items=np.array([7, 2, 7, 19, 0, 1], np.int64), device=device)
    for bad in ([20], [-1], [3, 25]):
        with pytest.raises(ValueError, match="outside"):
            aud.topk(ic, np.array(bad, np.int64))


def test_queries_ties_and_edges():
    run_queries()


# ---- the sliced sweep and the merge at the C ABI
def _p(t):
    return C.c_void_p(t.data_ptr())


def sliced_vs_unsliced(lib, ua, ia, excl, users, k, slices, device="cuda"):
    """mmssl_recommend_topk_sliced + mmssl_topk_merge == mmssl_recommend_topk, bitwise; the partial lists hold global ids of their
    own slice only, sorted by key."""
    n, I, d = users.size, ia.shape[0], ia.shape[1]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    ut, it, us, ip, ix = dev(ua), dev(ia), dev(users), dev(excl[0]), dev(excl[1])
    ref_ids = torch.empty(n, k, dtype=torch.int32, device=device)
    ref_sc = torch.empty(n, k, dtype=torch.float32, device=device)
    nb = lib.mmssl_recommend_workspace_bytes(n, k, I, d)
    ws = torch.zeros(max(nb // 8, 1), dtype=torch.int64, device=device)
    assert lib.mmssl_recommend_topk(_p(ut), d, _p(it), d, I, d, _p(us), n, _p(ip), _p(ix), k, k, _p(ref_ids), _p(ref_sc), _p(ws),
                                    None) == 0
    part_ids = torch.empty(slices, n, k, dtype=torch.int32, device=device)
    part_sc = torch.empty(slices, n, k, dtype=torch.float32, device=device)
    nb = lib.mmssl_recommend_sliced_workspace_bytes(n, k, I, d, slices)
    ws = torch.zeros(max(nb // 8, 1), dtype=torch.int64, device=device)
    assert lib.mmssl_recommend_topk_sliced(_p(ut), d, _p(it), d, I, d, _p(us), n, _p(ip), _p(ix), k, slices, _p(part_ids), _p(part_sc),
                                           _p(ws), None) == 0
    pi, ps = part_ids.cpu().numpy(), part_sc.cpu().numpy()
    for s in range(slices):
        lo, hi = I * s // slices, I * (s + 1) // slices
        real = pi[s] >= 0
        assert ((pi[s][real] >= lo) & (pi[s][real] < hi)).all()
        for r in range(n):
            m = int(real[r].sum())
            assert real[r, :m].all() and (ps[s, r, m:] == 0).all()
            key = host_key(ps[s, r, :m], pi[s, r, :m])
            assert (key[:-1] > key[1:]).all()
    out_ids = torch.full((n, k), -7, dtype=torch.int32, device=device)
    out_sc = torch.full((n, k), 7.0, dtype=torch.float32, device=device)
    assert lib.mmssl_topk_merge(_p(part_ids), _p(part_sc), n, slices, k, k, n * k, _p(out_ids), _p(out_sc), k, None) == 0
    assert torch.equal(out_ids.cpu(), ref_ids.cpu()) and np.array_equal(_bits(out_sc), _bits(ref_sc))
    return ref_ids, ref_sc


def slice_problem(I=300, U=11, d=8, seed=2):
    """Small-integer tables (exact, many equal scores) with a run of 40 identical candidate rows across several slice bounds, and
    exclusion rows of 0 to all candidates, dense around the bounds."""
    rng = np.random.default_rng(seed)
    ua = rng.integers(-2, 3, (U, d)).astype(np.float32)
    ia = rng.integers(-2, 3, (I, d)).astype(np.float32)
    ia[I // 3 - 20:I // 3 + 20] = ia[1]
    rows = [np.sort(rng.choice(I, size=int(rng.integers(0, I // 2)), replace=False)) for _ in range(U)]
    rows[3] = np.arange(I)
    rows[4] = np.arange(I // 3 - 30, I // 2 + 30)
    ip = np.zeros(U + 1, np.int64)
    np.cumsum([r.size for r in rows], out=ip[1:])
    users = np.array([4, 0, 3, 1, 2, 5, 6, 7, 8, 9, 10, 4], np.int64)
    return ua, ia, (ip, np.concatenate(rows).astype(np.int64)), users


def run_sliced(lib, k, slices, device="cuda"):
    ua, ia, excl, users = slice_problem()
    sliced_vs_unsliced(lib, ua, ia, excl, users, k, slices, device)


@pytest.mark.parametrize("k", [5, 70])
@pytest.mark.parametrize("slices", [1, 2, 3, 7, 301, 1000])
def test_sliced_equals_unsliced(k, slices):
    from mmssl_b200 import _lib
    run_sliced(_lib.load(require_device=True), k, slices)


def run_merge_model(lib, device="cuda", seed=0):
    """The merge against a host model: lists of random lengths whose scores include -0.0 / +0.0, exact ties across lists (told apart
    by id), NaN-free; the result does not depend on the order of the lists."""
    rng = np.random.default_rng(seed)
    n, P, k = 5, 6, 9
    pool = np.array([-0.0, 0.0, 1.0, -1.0, 2.5, -2.5, 1e-30, -1e-30], np.float32)
    ids = np.full((P, n, k), -1, np.int32)
    sc = np.zeros((P, n, k), np.float32)
    all_ids = rng.permutation(10 * P * k)[:P * n * k].reshape(P, n, k)
    for q in range(P):
        for r in range(n):
            m = int(rng.integers(0, k + 1)) if (q + r) % 4 else 0
            s = rng.choice(pool, m)
            key = host_key(s, all_ids[q, r, :m])
            o = np.argsort(key)[::-1]
            ids[q, r, :m], sc[q, r, :m] = all_ids[q, r, :m][o], s[o]
    results = []
    for perm in (np.arange(P), rng.permutation(P)):
        pi = torch.from_numpy(np.ascontiguousarray(ids[perm])).to(device)
        ps = torch.from_numpy(np.ascontiguousarray(sc[perm])).to(device)
        oi = torch.full((n, k + 3), -7, dtype=torch.int32, device=device)
        os_ = torch.full((n, k + 3), 7.0, dtype=torch.float32, device=device)
        assert lib.mmssl_topk_merge(_p(pi), _p(ps), n, P, k, k, n * k, _p(oi), _p(os_), k + 3, None) == 0
        results.append((oi.cpu().numpy(), os_.cpu().numpy()))
    for r in range(n):
        real = ids[:, r, :] >= 0
        kk = host_key(sc[:, r, :][real], ids[:, r, :][real])
        o = np.argsort(kk)[::-1][:k]
        want_i = np.full(k, -1, np.int32)
        want_s = np.zeros(k, np.float32)
        want_i[:o.size], want_s[:o.size] = ids[:, r, :][real][o], sc[:, r, :][real][o]
        for oi, os_ in results:
            assert np.array_equal(oi[r, :k], want_i) and np.array_equal(os_[r, :k].view(np.uint32), want_s.view(np.uint32)), r
            assert (oi[r, k:] == -7).all() and (os_[r, k:] == 7.0).all()
    assert any((sc.view(np.uint32) == 0x80000000).ravel())


def test_merge_against_host_model():
    from mmssl_b200 import _lib
    run_merge_model(_lib.load(require_device=True))


def run_forced_slices(monkeypatch, slices, device="cuda"):
    """Recommender and SimilarItems forced to slice: the evaluator's ranked lists / the unsliced lists, bit for bit."""
    from mmssl_b200 import recommend
    from mmssl_b200.similar import SimilarItems
    from tests.test_gpu_zz_recommend import run_against_evaluator
    ua, ia, train = problem(30, 700, 32, 9, n_excl=(0, 300))
    ic = torch.from_numpy(ia).to(device)
    plain = {k: SimilarItems(ic, k).topk(np.arange(0, 700, 3)) for k in (10, 80)}
    monkeypatch.setattr(recommend.Recommender, "_slices", lambda self, n: slices)
    for k in (10, 80):
        run_against_evaluator(30, 700, 32, k, 30, device=device, train=train, ua=ua, ia=ia)
        ids, sc = SimilarItems(ic, k).topk(np.arange(0, 700, 3))
        assert torch.equal(ids, plain[k][0]) and np.array_equal(_bits(sc), _bits(plain[k][1]))


@pytest.mark.parametrize("slices", [2, 5, 64])
def test_forced_slices_recommend_and_similar(monkeypatch, slices):
    run_forced_slices(monkeypatch, slices)


def run_slice_choice(device="cuda"):
    """The slice count the Recommender picks: 1 for a call that fills the GPU or a short candidate table, more for few queries
    against many candidates, bounded by the partial lists' memory; and the lists of a sliced call equal a forced unsliced one."""
    from mmssl_b200 import recommend
    rng = np.random.default_rng(1)
    U, I, d = 40000, 60, 32
    ua = rng.standard_normal((U, d)).astype(np.float32)
    ia = rng.standard_normal((I, d)).astype(np.float32)
    from mmssl_b200.audience import Audience
    aud = Audience.from_rows(torch.from_numpy(ua).to(device), {u: [u % I] for u in range(U)}, {}, {}, I, 20)
    rec = aud.rec
    assert rec._slices(8 * 2 * rec.sms) == 1 and rec._slices(1) > 1 and rec._slices(1) <= U // 4096
    items = np.array([3, 0, 59], np.int64)
    ic = torch.from_numpy(ia).to(device)
    got = aud.topk(ic, items)
    rec._slices = lambda n: 1
    want = aud.topk(ic, items)
    assert torch.equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1]))


def test_slice_choice():
    run_slice_choice()


@pytest.mark.parametrize("k", [20, 100])
@pytest.mark.parametrize("name", ["baby", "sports"])
def test_dataset_shape_sliced_equals_unsliced(name, k):
    """Few items against every user of Baby / Sports: the sliced call (the Recommender's choice) == the unsliced one, bitwise."""
    from mmssl_b200.audience import Audience
    U, I, d, ua, ia, train = _config(name)
    aud = Audience.from_rows(torch.from_numpy(ua).cuda(), train, {}, {}, I, k)
    ic = torch.from_numpy(ia).cuda()
    items = np.array([5, 0, I - 1, 77, 5, 1000, 2], np.int64)
    assert aud.rec._slices(items.size) > 1
    got = aud.topk(ic, items)
    aud.rec._slices = lambda n: 1
    want = aud.topk(ic, items)
    assert torch.equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1]))


def run_sharded_one_process(tmp_path, exclude, U=53, I=31, d=8, device="cuda"):
    """Both ranks of a world-2 ShardedAudience in one process, chunk by chunk: each rank ranks the chunk against its user block,
    then a stand-in for the all-to-all hands each rank the rows every rank sent it, and the rank merges them.  The lists of each
    rank's items == the one-GPU Audience, bitwise, for a user count that is not a multiple of the world size and an item list
    that rank 0 owns none of."""
    from mmssl_b200 import audience
    from mmssl_b200.parallel import RowPartition
    assert U % 2
    ua, ia, train = problem(U, I, d, 8, n_excl=(0, 12))
    rng = np.random.default_rng(8)
    test = {u: rng.choice(I, size=2, replace=False).tolist() for u in range(U)}
    val = {u: rng.choice(I, size=1, replace=False).tolist() for u in range(0, U, 2)}
    pu, pi = RowPartition(U, 2), RowPartition(I, 2)
    uc, ic = torch.from_numpy(ua).to(device), torch.from_numpy(ia).to(device)
    one = audience.Audience.from_rows(uc, train, test, val, I, 7, exclude)
    k = 7
    for name, items in (("all", rng.permutation(I)), ("rank1_only", np.arange(pi.block, I)[::-1].copy())):
        ranks = [audience.ShardedAudience.from_rows(train, test, val, U, I, pu, pi, r, k, exclude, device=device) for r in range(2)]
        recs = [ranks[r].local(pu.local(uc, r)) for r in range(2)]
        got = {0: [], 1: []}
        for s in range(0, items.size, 4):                   # chunks of 4; per chunk both ranks send before either merges
            c = items[s:s + 4]
            sent = {}
            for r in range(2):
                def capture(send, send_rows, recv_rows, r=r):
                    sent[r] = (send.clone(), list(send_rows))
                    return torch.full((int(sum(recv_rows)), 2 * k), -1, dtype=torch.int32, device=device)
                ranks[r].exchange = capture
                ranks[r]._chunk(recs[r], ic, c)
            for r in range(2):
                def deliver(send, send_rows, recv_rows, r=r):
                    blocks = []
                    for src in range(2):
                        buf, rows = sent[src]
                        off = int(sum(rows[:r]))
                        blocks.append(buf[off:off + rows[r]])
                    return torch.cat(blocks)
                ranks[r].exchange = deliver
                got[r].append(ranks[r]._chunk(recs[r], ic, c))
        assert items[ranks[0].mine(items)].size == (0 if name == "rank1_only" else items[items < pi.block].size)
        for r in range(2):
            mine = items[ranks[r].mine(items)]
            gi = torch.cat([g[0] for g in got[r]]).to(torch.int64)
            gs = torch.cat([g[1] for g in got[r]])
            wi, ws = one.topk(ic, mine)
            assert torch.equal(gi.cpu(), wi.cpu()) and np.array_equal(_bits(gs), _bits(ws)), (name, r)
    return one, uc, ic


@pytest.mark.parametrize("exclude", ["train", "seen"])
def test_sharded_one_process(tmp_path, exclude):
    run_sharded_one_process(tmp_path, exclude)


def run_trainer(tmp_path, device="cuda", epochs=2):
    """Trainer.audience after training, and on a fresh Trainer that loaded the checkpoint: the same lists; every (item, user,
    score) of an audience list has the bits of the score Trainer.recommend gives the pair where it lists it."""
    from tests.test_gpu_zz_recommend import trainer
    ckpt = str(tmp_path / "run.ckpt")
    tr = trainer(device, epochs=epochs, ckpt=ckpt)
    tr.train()
    items = np.arange(tr.n_items)
    for exclude in ("train", "seen"):
        ids, sc = tr.audience(items, 8, exclude)
        fresh = trainer(device, epochs=epochs)
        fresh.load(ckpt)
        ids2, sc2 = fresh.audience(items, 8, exclude)
        assert torch.equal(ids, ids2) and np.array_equal(_bits(sc), _bits(sc2))
        r_ids, r_sc = tr.recommend(np.arange(tr.n_users), tr.n_items, exclude)
        r_ids, r_sc = r_ids.cpu().numpy(), r_sc.cpu().numpy()
        ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
        found = 0
        for i in range(tr.n_items):
            for u, s in zip(ids[i], sc[i]):
                if u < 0:
                    continue
                at = np.nonzero(r_ids[u] == i)[0]
                assert at.size == 1, (i, u)
                assert r_sc[u, at[0]].view(np.uint32) == np.float32(s).view(np.uint32), (i, u)
                found += 1
        assert found > 0


def test_trainer_audience(tmp_path):
    run_trainer(tmp_path)
