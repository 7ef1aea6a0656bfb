"""Evaluation with any cut-off list (``mmssl_eval_rank_wide``: more than 8 cut-offs, K > 64, K >= n_items) against the
oracle on the kernel's own scores, the golden vectors minted from the reference with wide Ks
(tests/golden/make_golden_eval_wide.py) and the <= 64 path on the same inputs."""
import os

import numpy as np
import pytest
import torch

from oracle import eval_oracle as EO
from tests import eval_full_oracle as FO
from tests.test_gpu_zz_eval import _rows
from tests.test_gpu_zz_eval_full import _csr

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["eval_wide_random", "eval_wide_ties", "eval_wide_short", "eval_wide_full"]


def _bits(t):
    return t.cpu().numpy().view(np.uint8)


def check_against_oracle(ev, ua, ia, users, g_train, g_held, Ks, is_val):
    """ranked / hits exactly the oracle's on the kernel's scores, per_user / result / AUC within 1e-12, a second run bitwise
    equal, and in full mode the AUC bitwise equal to what the <= 64 path computes."""
    from mmssl_b200.evaluate import Evaluator
    assert ev.wide
    uc, ic = torch.from_numpy(ua).cuda(), torch.from_numpy(ia).cuda()
    out = ev.rank(uc, ic, users, is_val, want_scores=True)
    torch.cuda.synchronize()
    s_gpu = out["scores"].cpu().numpy()
    ref = EO.evaluate(ua, ia, users, g_train[0], g_train[1], g_held[0], g_held[1], Ks, rating=s_gpu)
    assert out["ranked"].shape == (len(users), max(Ks))
    assert np.array_equal(out["ranked"].cpu().numpy().astype(np.int64), ref["ranked"])
    assert np.array_equal(out["hits"].cpu().numpy().astype(np.int64), ref["hits"])
    np.testing.assert_allclose(out["per_user"].cpu().numpy(), ref["per_user"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(out["result"].cpu().numpy(), ref["result"], rtol=0, atol=1e-12)
    top, sc = out["ranked"].cpu().numpy(), out["ranked_scores"].cpu().numpy()
    for n in range(len(users)):
        m = int((top[n] >= 0).sum())
        assert np.array_equal(sc[n, :m], s_gpu[n, top[n, :m]])
    again = ev.rank(uc, ic, users, is_val)
    for k in ("ranked", "ranked_scores", "hits", "per_user", "result") + (("auc",) if "auc" in out else ()):
        assert np.array_equal(_bits(again[k]), _bits(out[k])), k
    if "auc" in out:
        fo = FO.evaluate(ua, ia, users, g_train[0], g_train[1], g_held[0], g_held[1], Ks, rating=s_gpu)
        auc = out["auc"].cpu().numpy()
        assert np.array_equal(np.isnan(auc), np.isnan(fo["auc_per_user"]))
        np.testing.assert_allclose(auc, fo["auc_per_user"], rtol=0, atol=1e-12)
        narrow = Evaluator(ev._train_rows, ev._held_rows[False], ev._held_rows[True], ev.n_users, ev.n_items, [10],
                           device=ev.device, test_flag="full")
        assert np.array_equal(_bits(narrow.rank(uc, ic, users, is_val)["auc"]), _bits(out["auc"]))
    return out


class _Ev:
    """Evaluator that remembers its rows, so a twin with other Ks can be built from the same input."""

    def __new__(cls, train, test, val, U, I, Ks, test_flag="part"):
        from mmssl_b200.evaluate import Evaluator
        ev = Evaluator(train, test, val, U, I, Ks, test_flag=test_flag)
        ev._train_rows, ev._held_rows = train, {False: test, True: val}
        return ev


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("split", ["test", "val"])
def test_eval_wide_matches_reference_golden(case, split):
    g = np.load(os.path.join(GOLD, case + ".npz"))
    Ks = [int(k) for k in g["Ks"]]
    U, I = g["ua"].shape[0], g["ia"].shape[0]
    flag = "full" if case == "eval_wide_full" else "part"
    ev = _Ev(_rows(g["train_indptr"], g["train_indices"]), _rows(g["test_indptr"], g["test_indices"]),
             _rows(g["val_indptr"], g["val_indices"]), U, I, Ks, test_flag=flag)
    users = g[f"{split}_users"]
    held = (g[f"{split}_indptr"], g[f"{split}_indices"])
    out = check_against_oracle(ev, g["ua"], g["ia"], users, (g["train_indptr"], g["train_indices"]), held, Ks, split == "val")
    if case in ("eval_wide_ties", "eval_wide_full"):
        # quantised embeddings: every score is exact in fp32 whatever the summation order, so the reference's own results
        assert np.array_equal(out["ranked"].cpu().numpy().astype(np.int64), g[f"{split}_ranked"])
        assert np.array_equal(out["hits"].cpu().numpy().astype(np.int64), g[f"{split}_hits"])
        np.testing.assert_allclose(out["per_user"].cpu().numpy(), g[f"{split}_per_user"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(out["result"].cpu().numpy(), g[f"{split}_result"], rtol=0, atol=1e-12)
    res = ev.test_torch(torch.from_numpy(g["ua"]).cuda(), torch.from_numpy(g["ia"]).cuda(), list(users), split == "val")
    assert set(res) == {"precision", "recall", "ndcg", "hit_ratio", "auc"} and res["recall"].shape == (len(Ks),)


def run_consistency_with_narrow(U=300, I=2500, d=32, seed=4, full=False):
    """Ks = [10, 20, 50, 100] (wide path) against [10, 20, 50] (<= 64 path): the first 50 columns of ranked / hits and
    precision, recall, hit at 10 / 20 / 50 bitwise equal; ndcg differs (the ideal DCG sees the hits at ranks 50..99)
    and matches the oracle (checked inside check_against_oracle)."""
    rng = np.random.default_rng(seed)
    ua = rng.standard_normal((U, d)).astype(np.float32)
    ia = rng.standard_normal((I, d)).astype(np.float32)
    train = {u: sorted(rng.choice(I, size=int(rng.integers(0, 200)), replace=False).tolist()) for u in range(U)}
    train = {u: v for u, v in train.items() if v}
    held = {u: rng.choice(I, size=int(rng.integers(1, 120)), replace=False).tolist() for u in range(U)}
    flag = "full" if full else "part"
    wide = _Ev(train, held, {}, U, I, [10, 20, 50, 100], test_flag=flag)
    users = rng.permutation(U).astype(np.int64)
    out = check_against_oracle(wide, ua, ia, users, _csr(train, U), _csr(held, U), [10, 20, 50, 100], False)
    from mmssl_b200.evaluate import Evaluator
    narrow = Evaluator(train, held, {}, U, I, [10, 20, 50], test_flag=flag)
    assert not narrow.wide
    no = narrow.rank(torch.from_numpy(ua).cuda(), torch.from_numpy(ia).cuda(), users, False)
    for k in ("ranked", "ranked_scores", "hits"):
        assert np.array_equal(_bits(out[k][:, :50].contiguous()), _bits(no[k])), k
    pw, pn = out["per_user"].cpu().numpy(), no["per_user"].cpu().numpy()
    for metric in (0, 1, 3):
        assert np.array_equal(pw[:, metric, :3].view(np.uint64), pn[:, metric, :].view(np.uint64)), metric
    assert not np.array_equal(pw[:, 2, :3], pn[:, 2, :])              # the quirk shows: some ndcg@K moved
    if full:
        assert np.array_equal(_bits(out["auc"]), _bits(no["auc"]))


def test_eval_wide_consistent_with_narrow_part():
    run_consistency_with_narrow()


def test_eval_wide_consistent_with_narrow_full():
    run_consistency_with_narrow(full=True)


def _baby():
    from mmssl_b200.synthetic import CONFIGS, make_bipartite
    U, I, nnz, d, *_ = CONFIGS["baby"]
    tr = make_bipartite(U, I, nnz, seed=3).tocsr()
    tr.sort_indices()
    rng = np.random.default_rng(2)
    held = {u: rng.choice(I, size=int(rng.integers(1, 9)), replace=False).tolist() for u in range(U)}
    ua = rng.standard_normal((U, d)).astype(np.float32)
    ia = rng.standard_normal((I, d)).astype(np.float32)
    train_rows = {u: tr.indices[tr.indptr[u]:tr.indptr[u + 1]].tolist() for u in range(U) if tr.indptr[u + 1] > tr.indptr[u]}
    return U, I, ua, ia, train_rows, held, (tr.indptr.astype(np.int64), tr.indices.astype(np.int64))


@pytest.mark.parametrize("Ks", [[10, 20, 50, 100, 1000], [7050]])
@pytest.mark.parametrize("flag", ["part", "full"])
def test_eval_wide_baby_size(Ks, flag):
    """Every Baby-size user (19445 x 7050, d = 64), part and full mode; max(Ks) = 1000 and max(Ks) = n_items both use the
    global workspace, with several tiles per CTA."""
    U, I, ua, ia, train_rows, held, g_train = _baby()
    assert I == 7050
    ev = _Ev(train_rows, held, {}, U, I, Ks, test_flag=flag)
    check_against_oracle(ev, ua, ia, np.arange(U, dtype=np.int64), g_train, _csr(held, U), Ks, False)


def run_trainer_wide(device="cuda"):
    """A Trainer life cycle with Ks = [10, 20, 50, 100]: test() returns 4-column results equal to a fresh Evaluator's."""
    from mmssl_b200.dataset import ReferenceDataset
    from mmssl_b200.evaluate import Evaluator
    from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed
    ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
    args = TrainerArgs(dataset="dataset_small", epoch=1, batch_size=16, verbose=1, early_stopping_patience=1, m_topk_rate=0.05,
                       Ks="[10, 20, 50, 100]", seed=5)
    set_seed(args.seed)
    tr = Trainer(ds, args, device=device, log=None)
    _, test_ret = tr.train()
    assert test_ret is not None and test_ret["recall"].shape == (4,)
    users = sorted(ds.test_set)
    ret = tr.test(users, is_val=False)
    hs = tr.step.hs
    outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, None, want_sumsq=False)
    ev = Evaluator(ds.train_items, ds.test_set, ds.val_set, tr.n_users, tr.n_items, tr.Ks, device=device)
    want = ev.test_torch(outs[0], outs[1], users, False)
    for k in ("precision", "recall", "ndcg", "hit_ratio"):
        assert ret[k].shape == (4,) and np.array_equal(ret[k], want[k]), k


def test_trainer_wide_ks():
    run_trainer_wide()


def run_rejected_input(device="cuda"):
    from mmssl_b200.evaluate import Evaluator
    rows = {0: [1], 1: [2]}
    for Ks in ([0], [], [10, 0, 100], [-5]):
        with pytest.raises(ValueError):
            Evaluator(rows, rows, {}, 2, 5, Ks, device=device)
    assert Evaluator(rows, rows, {}, 2, 5, [1000], device=device).wide


def test_rejected_input():
    run_rejected_input()
