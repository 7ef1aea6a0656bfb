"""Fold-in (mmssl_fold_users through mmssl_b200/foldin.py) on the H100.
  * against float64: seeded tables at every width and K = 1, 2, 3, query rows of degree 0, 1, 63, 64, 65, 1024, 1025, 5000 and one
    holding every item, with and without id rows -- per row within K_FP32 times the distance of the same restatement in fp32;
  * identity with the forward: every user's own training row, folded with its id, is bitwise the forward's u_f row up to the
    SpMM's heavy cut (empty rows too) and within the fp64 bound above it, with empty and with non-empty modality graphs;
  * batch invariance and determinism: a query's row and list alone, among 10^4 others, duplicated, and from call to call;
  * semantics: query items never listed, "train" / "seen" for id queries only, a row holding every item, duplicates, refusals;
  * the export round trip and the four readers' refusals; one process holding both ranks of a world-2 ShardedFoldIn;
  * Trainer.recommend_for == Trainer.recommend on the training rows, the same after Trainer.load, no effect on the next step.
The bodies also run on the CPU emulator (tests/test_emu_foldin.py)."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.test_gpu_zz_recommend import _bits

pytestmark = pytest.mark.gpu
K_FP32 = 4.0
FLOOR = 8 * 2.0 ** -24          # a few fp32 roundings of the combine: where the fp32 restatement happens to land on float64
CUTS = (64, 32, 1024, 64)       # csrc/graph.cu: split threshold, segment, heavy threshold, heavy segment


# ------------------------------------------------------------------ 1. against float64
def restate(q, users, u0, layers, xv, xt, rate, dt):
    """The fold-in contract in dtype dt on the given fp32 inputs: sequential sums in the row's order, a long row cut into the
    plan's segments whose sums are added in order, softmax on the last layer, the forward's running sum and combine."""
    from mmssl_b200.foldin import row_weights
    ip, ix = q
    K, d = len(layers), xv.shape[1]
    w = row_weights(np.diff(ip)).astype(dt)
    out = np.zeros((ip.size - 1, d), dt)

    def rsum(t, r):
        rows = t[ix[ip[r]:ip[r + 1]]].astype(dt)
        n = rows.shape[0]
        if n == 0:
            return np.zeros(d, dt)
        if n <= CUTS[0]:
            return np.cumsum(w[r] * rows, axis=0, dtype=dt)[-1]
        sl = CUTS[1] if n <= CUTS[2] else CUTS[3]
        segs = [np.cumsum(w[r] * rows[s:s + sl], axis=0, dtype=dt)[-1] for s in range(0, n, sl)]
        return np.cumsum(np.array(segs, dt), axis=0, dtype=dt)[-1]

    def unit(v):
        return v / max(np.sqrt(np.sum(v * v, dtype=dt)), dt(1e-12))

    for r in range(ip.size - 1):
        s = u0[users[r]].astype(dt) if users[r] >= 0 else np.zeros(d, dt)
        for k in range(K):
            v = rsum(layers[k], r)
            if k == K - 1:
                e = np.exp(v - v.max())
                v = e / np.sum(e, dtype=dt)
            s = s + v
        out[r] = s * dt(1.0 / (K + 1)) + dt(rate) * (unit(rsum(xv, r)) + unit(rsum(xt, r)))
    return out


def degree_rows(I, degs, seed):
    rng = np.random.default_rng(seed)
    rows = [np.sort(rng.choice(I, size=min(g, I), replace=False)) for g in degs]
    ip = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([r.size for r in rows], out=ip[1:])
    return ip, np.concatenate(rows).astype(np.int64)


def run_fp64(d, K, I=6000, degs=(0, 1, 63, 64, 65, 1024, 1025, 5000, 6000), U=50, device="cuda", seed=0):
    from mmssl_b200.foldin import FoldIn
    rng = np.random.default_rng(seed + 10 * d + K)
    layers = [rng.standard_normal((I, d)).astype(np.float32) for _ in range(K)]
    xv, xt = (rng.standard_normal((I, d)).astype(np.float32) for _ in range(2))
    items = rng.standard_normal((I, d)).astype(np.float32)
    u0 = rng.standard_normal((U, d)).astype(np.float32)
    dev = lambda a: torch.from_numpy(a).to(device)
    fi = FoldIn(dev(u0), [dev(t) for t in layers], dev(xv), dev(xt), dev(items), 0.55)
    q = degree_rows(I, degs, seed)
    n = q[0].size - 1
    for users in (np.full(n, -1, np.int64), rng.integers(0, U, n).astype(np.int64)):
        got = fi.fold(q, users).cpu().numpy().astype(np.float64)
        f64 = restate(q, users, u0, layers, xv, xt, 0.55, np.float64)
        f32 = restate(q, users, u0, layers, xv, xt, 0.55, np.float32).astype(np.float64)
        for r in range(n):
            nrm = np.linalg.norm(f64[r])
            e_dev, e_32 = np.linalg.norm(got[r] - f64[r]) / nrm, np.linalg.norm(f32[r] - f64[r]) / nrm
            assert e_dev <= max(K_FP32 * e_32, FLOOR), (d, K, degs[r], users[r], e_dev, e_32)
    return fi


@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("d", [32, 64, 96, 128, 192, 256])
def test_against_float64(d, K):
    run_fp64(d, K)


# ------------------------------------------------------------------ 2. identity with the forward
def model(U, I, d, K, fused, device, seed=1):
    """A seeded model on a synthetic graph: users of degree 0, 1..63, 64, 65, 100, 1024, 1025, 1500 (the SpMM's cuts), items
    with the rest; modality graphs empty or random."""
    from mmssl_b200.engine import Engine, FeatureStore
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.synthetic import csr_norm
    rng = np.random.default_rng(seed)
    degs = np.concatenate([[0, 0, 1, 63, 64, 65, 100, 1024, 1025, 1500], rng.integers(1, 40, U - 10)])
    rows = [np.sort(rng.choice(I, size=g, replace=False)) for g in degs]
    R = sp.csr_matrix((np.ones(int(degs.sum()), np.float32), np.concatenate(rows), np.concatenate([[0], np.cumsum(degs)])),
                      shape=(U, I))
    R.sort_indices()
    G = lambda m: BipartiteGraph.from_scipy(m, device=device)
    if fused:
        M = sp.random(U, I, density=0.02, random_state=seed, format="csr", dtype=np.float32)
        M.data[:] = 1
        mod = [G(csr_norm(M)), G(csr_norm(M.T.tocsr()))]
        graphs = (G(csr_norm(R)), G(csr_norm(R.T.tocsr())), mod[0], mod[1], mod[0], mod[1])
    else:
        empty = sp.csr_matrix((U, I), dtype=np.float32)
        graphs = (G(csr_norm(R)), G(csr_norm(R.T.tocsr())), G(empty), G(empty.T.tocsr()), G(empty), G(empty.T.tocsr()))
    Dv, Dt = 24, 16
    f = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32) * 0.3).to(device)
    P = {"image_trans.weight": f(d, Dv), "image_trans.bias": f(d), "text_trans.weight": f(d, Dt), "text_trans.bias": f(d),
         "user_id_embedding.weight": f(U, d), "item_id_embedding.weight": f(I, d), "weight_dict.w_self_attention_cat": f(4 * d, d)}
    feats = (FeatureStore(f(I, Dv)), FeatureStore(f(I, Dt)))
    return Engine(d, K), P, feats, graphs, R


def run_identity(d, K, fused, U=300, I=2000, device="cuda"):
    """Every user's training row, folded with its id, against the u_f row of the same forward whose tables it folds from."""
    from mmssl_b200.foldin import FoldIn
    eng, P, feats, graphs, R = model(U, I, d, K, fused, device)
    outs, st = eng.forward(P, feats, graphs, None, want_sumsq=False, keep_fold=True)
    assert st.fused == fused and len(st.i_layers) == K
    fi = FoldIn(st.u0, st.i_layers, st.X2[:, :d], st.X2[:, d:], outs[1], eng.cat_rate)
    users = np.arange(U, dtype=np.int64)
    got = fi.fold((R.indptr.astype(np.int64), R.indices.astype(np.int64)), users).cpu().numpy()
    want = outs[0].cpu().numpy()
    deg = np.diff(R.indptr)
    light = deg <= CUTS[2]
    assert np.array_equal(_bits(got[light]), _bits(want[light])), np.nonzero((got != want).any(1) & light)[0]
    heavy = np.nonzero(~light)[0]                # the forward sums these with float atomics: both within check 1's bound
    if heavy.size:
        np_ = lambda t: t.detach().cpu().numpy()
        q = (np.concatenate([[0], np.cumsum(deg[heavy])]).astype(np.int64),
             np.concatenate([R.indices[R.indptr[u]:R.indptr[u + 1]] for u in heavy]).astype(np.int64))
        args = (q, heavy, np_(st.u0), [np_(t) for t in st.i_layers], np_(st.X2[:, :d]), np_(st.X2[:, d:]), eng.cat_rate)
        f64, f32 = restate(*args, np.float64), restate(*args, np.float32).astype(np.float64)
        for j, u in enumerate(heavy):
            nrm = np.linalg.norm(f64[j])
            bound = max(K_FP32 * np.linalg.norm(f32[j] - f64[j]) / nrm, FLOOR)
            for row in (got[u], want[u]):
                assert np.linalg.norm(row.astype(np.float64) - f64[j]) / nrm <= bound, u
    return eng, P, feats, graphs, R, fi


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("d,K", [(64, 2), (32, 1), (96, 3), (128, 2), (192, 1), (256, 3)])
def test_identity_with_forward(d, K, fused):
    run_identity(d, K, fused)


# ------------------------------------------------------------------ 3. batch invariance and determinism
def run_invariance(n_others=10000, device="cuda"):
    from mmssl_b200.foldin import FoldIn
    fi = run_fp64(64, 2, I=1500, degs=(3,), device=device)
    rng = np.random.default_rng(4)
    degs = np.concatenate([[0, 1, 65, 1100], rng.integers(0, 40, n_others)])
    q = degree_rows(1500, degs, 5)
    users = np.where(rng.random(degs.size) < 0.5, rng.integers(0, fi.n_users, degs.size), -1).astype(np.int64)
    probe = [0, 1, 2, 3, 7]
    alone = {p: (fi.fold(sub(q, [p]), users[[p]]), fi.topk(sub(q, [p]), 12, users[[p]])) for p in probe}
    order = rng.permutation(degs.size)
    qq, uu = sub(q, order), users[order]
    many = fi.fold(qq, uu)
    ids, sc = fi.topk(qq, 12, uu)
    ids2, sc2 = fi.topk(qq, 12, uu)
    assert torch.equal(ids, ids2) and np.array_equal(_bits(sc), _bits(sc2))
    dup = sub(q, probe + probe[::-1])
    dup_rows = fi.fold(dup, users[probe + probe[::-1]])
    for j, p in enumerate(probe):
        at = int(np.nonzero(order == p)[0][0])
        row, (li, ls) = alone[p]
        assert np.array_equal(_bits(many[at]), _bits(row[0])), p
        assert torch.equal(ids[at], li[0]) and np.array_equal(_bits(sc[at]), _bits(ls[0])), p
        assert np.array_equal(_bits(dup_rows[j]), _bits(row[0])) and np.array_equal(_bits(dup_rows[len(probe) * 2 - 1 - j]), _bits(row[0]))


def sub(q, pick):
    ip, ix = q
    rows = [ix[ip[p]:ip[p + 1]] for p in pick]
    out = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([r.size for r in rows], out=out[1:])
    return out, (np.concatenate(rows) if rows else np.zeros(0, np.int64))


def test_batch_invariance_and_determinism():
    run_invariance()


# ------------------------------------------------------------------ 4. semantics
def run_semantics(tmp_path, device="cuda"):
    from mmssl_b200 import audience, foldin, recommend, similar
    from mmssl_b200.foldin import FoldIn
    I, U, d = 300, 20, 32
    rng = np.random.default_rng(7)
    dev = lambda a: torch.from_numpy(a).to(device)
    t = lambda: dev(rng.standard_normal((I, d)).astype(np.float32))
    train = foldin.prepare_rows(degree_rows(I, rng.integers(1, 30, U), 8), I)
    val = foldin.prepare_rows(degree_rows(I, rng.integers(0, 4, U), 9), I)
    test = foldin.prepare_rows(degree_rows(I, rng.integers(0, 4, U), 10), I)
    fi = FoldIn(dev(rng.standard_normal((U, d)).astype(np.float32)), [t(), t()], t(), t(), t(), 0.55, held=(train, val, test))
    q = degree_rows(I, [5, 0, 17, I, 2], 11)
    users = np.array([3, 4, -1, -1, 3], np.int64)
    k = I
    for ex in ("train", "seen"):
        ids, _ = fi.topk(q, k, users, ex)
        ids = ids.cpu().numpy()
        for r in range(users.size):
            bar = set(q[1][q[0][r]:q[0][r + 1]].tolist())
            if users[r] >= 0:
                for h in ((train,) if ex == "train" else (train, val, test)):
                    bar |= set(h[1][h[0][users[r]]:h[0][users[r] + 1]].tolist())
            got = ids[r][ids[r] >= 0]
            assert set(got.tolist()) == set(range(I)) - bar, (ex, r)
        assert (ids[3] == -1).all()                   # a row holding every item
    # duplicates count once, in any order
    a = fi.fold((np.array([0, 3]), np.array([5, 9, 2])))
    b = fi.fold((np.array([0, 6]), np.array([9, 2, 5, 5, 9, 2])))
    assert np.array_equal(_bits(a), _bits(b))
    # refusals
    for bad in ((np.array([0, 1]), np.array([I])), (np.array([0, 1]), np.array([-1]))):
        with pytest.raises(ValueError, match="outside"):
            fi.fold(bad)
    for bad_u in ([U], [-2]):
        with pytest.raises(ValueError, match="users"):
            fi.fold((np.array([0, 1]), np.array([1])), np.array(bad_u))
    with pytest.raises(ValueError, match="width"):
        FoldIn(None, [t()], t(), dev(np.zeros((I, 64), np.float32)), t())
    with pytest.raises(ValueError, match="at most"):
        FoldIn(None, [t()] * (foldin.MAX_LAYERS + 1), t(), t(), t())
    with pytest.raises(ValueError, match="exclude"):
        fi.topk(q, 3, users, "all")
    # export -> read round trip, chunked; the readers refuse each other's formats
    want_ids, want_sc = fi.topk(q, 7, users, "seen")
    out = str(tmp_path / "fold")
    assert fi.export(q, 7, out, users, "seen", chunk=2) == users.size
    qs, ids, sc = foldin.read(out)
    assert np.array_equal(qs, np.arange(users.size)) and np.array_equal(ids, want_ids.cpu().numpy())
    assert np.array_equal(_bits(sc), _bits(want_sc))
    for other in (recommend.read, similar.read, audience.read):
        with pytest.raises(ValueError, match="fold-in"):
            other(out)
    rec = recommend.Recommender(t(), (dev(np.zeros(U + 1, np.int64)), dev(np.zeros(1, np.int64))), 3)
    rdir = str(tmp_path / "rec")
    rec.export(dev(rng.standard_normal((U, d)).astype(np.float32)), np.arange(U), rdir)
    with pytest.raises(ValueError, match="recommendations"):
        foldin.read(rdir)
    return fi


def test_semantics(tmp_path):
    run_semantics(tmp_path)


def run_sharded_one_process(device="cuda"):
    """Both ranks of a world-2 ShardedFoldIn in one process on the gathered tables: each rank's lists are the one-GPU FoldIn's,
    bitwise, for its own id queries and for new users; a user of the other rank is refused."""
    from mmssl_b200.foldin import FoldIn, ShardedFoldIn
    from mmssl_b200.parallel import RowPartition
    U, I, d = 21, 200, 64
    rng = np.random.default_rng(12)
    dev = lambda a: torch.from_numpy(a).to(device)
    t = lambda n: dev(rng.standard_normal((n, d)).astype(np.float32))
    from mmssl_b200.foldin import prepare_rows
    train = prepare_rows(degree_rows(I, rng.integers(1, 20, U), 13), I)
    u0, tabs = t(U), [t(I) for _ in range(5)]
    one = FoldIn(u0, tabs[:2], tabs[2], tabs[3], tabs[4], 0.55, held=(train,) * 3)
    pu = RowPartition(U, 2)
    q = degree_rows(I, rng.integers(0, 30, 9), 14)
    for r in range(2):
        lo, hi = pu.bounds(r)
        held = tuple((train[0][lo:hi + 1] - train[0][lo], train[1][train[0][lo]:train[0][hi]]) for _ in range(3))
        held = tuple((np.concatenate([h[0], np.full(pu.block - (hi - lo), h[0][-1])]), h[1]) for h in held)
        sh = ShardedFoldIn(FoldIn(pu.local(u0, r), tabs[:2], tabs[2], tabs[3], tabs[4], 0.55, held), pu, r)
        users = np.where(np.arange(9) % 3 == 0, -1, rng.integers(lo, hi, 9)).astype(np.int64)
        got = sh.topk(q, 9, users, "train")
        want = one.topk(q, 9, users, "train")
        assert torch.equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1])), r
        assert np.array_equal(_bits(sh.fold(q, users)), _bits(one.fold(q, users)))
        assert np.array_equal(sh.mine(np.array([lo, hi - 1, -1, (lo + pu.block) % U])), [0, 1])
        with pytest.raises(ValueError, match="not held by rank"):
            sh.topk(q, 3, np.full(9, (lo + pu.block) % U))


def test_sharded_one_process():
    run_sharded_one_process()


# ------------------------------------------------------------------ Trainer
def run_trainer(tmp_path, device="cuda", k=10):
    """recommend_for on every user's training row with its id == recommend, bitwise, for both exclusion sets; the same lists
    after Trainer.load; fold_in / recommend_for leave the next training step bitwise unchanged."""
    from mmssl_b200.dataset import held_csr
    from tests.test_gpu_zz_recommend import trainer
    path = str(tmp_path / "run.ckpt")
    tr = trainer(device, epochs=1, ckpt=path)
    tr.train()
    # the users whose train.json row is their row of the training matrix (the small dataset has one that is not: its training
    # row folds to its u_f, but recommend excludes the train.json row)
    R = tr.ui_graph_raw
    items = tr.data.train_items
    users = np.array([u for u in range(tr.n_users) if sorted(set(items.get(u, []))) == R.indices[R.indptr[u]:R.indptr[u + 1]].tolist()],
                     np.int64)
    assert users.size >= tr.n_users - 1
    rows = held_csr({int(u): items.get(int(u), []) for u in users}, tr.n_users)
    rows = (np.concatenate([[0], np.cumsum(np.diff(rows[0])[users])]), rows[1])
    for ex in ("train", "seen"):
        ids, sc = tr.recommend_for(rows, k, users, ex)
        want_ids, want_sc = tr.recommend(users, k, ex)
        assert torch.equal(ids, want_ids) and np.array_equal(_bits(sc), _bits(want_sc)), ex
    new = tr.recommend_for(rows, k)
    fresh = trainer(device, epochs=1)
    fresh.load(path)
    assert torch.equal(fresh.recommend_for(rows, k)[0], new[0]) and np.array_equal(_bits(fresh.recommend_for(rows, k)[1]), _bits(new[1]))
    # the next step: a twin loaded from the same checkpoint that does not fold
    twin = trainer(device, epochs=1)
    twin.load(path)
    from mmssl_b200 import checkpoint
    state = checkpoint.rng_state(device)
    fresh.fold_in(rows, users)
    fresh.recommend_for(rows, k, users, "seen")
    after = checkpoint.rng_state(device)
    assert torch.equal(after["torch"], state["torch"]) and after["random"] == state["random"]      # no RNG draws
    assert all(torch.equal(after[g], state[g]) for g in ("cuda",) if g in state)
    us = sorted(tr.data.train_items)[:tr.batch_size]
    batch = (us, [int(tr.data.train_items[u][0]) for u in us], [(5 + j) % tr.n_items for j in range(len(us))])
    fresh.step.step(*batch)
    checkpoint.set_rng_state(state, device)         # the twin's step draws what the first one drew
    twin.step.step(*batch)
    for name in fresh.P:
        assert np.array_equal(_bits(fresh.P[name]), _bits(twin.P[name])), name


def test_trainer(tmp_path):
    run_trainer(tmp_path)
