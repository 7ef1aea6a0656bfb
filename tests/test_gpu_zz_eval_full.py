"""Full-mode evaluation on the device (``Evaluator(..., test_flag='full')`` -> mmssl_eval_rank_full): per-user ROC-AUC
against the oracle on the kernel's own scores and against the golden vectors minted from the reference's
``--test_flag full`` run; the ranking outputs are those of part mode, bit for bit."""
import os

import numpy as np
import pytest
import torch

from tests import eval_full_oracle as FO
from tests.test_gpu_zz_eval import _rows

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["eval_full_random", "eval_full_ties", "eval_full_short", "eval_full_edges"]


def _same_nan(a, b):
    assert np.array_equal(np.isnan(a), np.isnan(b))


def _csr(rows, U):
    ptr = np.zeros(U + 1, np.int64)
    for u in range(U):
        ptr[u + 1] = ptr[u] + len(rows.get(u, []))
    idx = np.concatenate([np.sort(np.asarray(rows.get(u, []), np.int64)) for u in range(U)]) if ptr[-1] else np.zeros(0, np.int64)
    return ptr, idx


def check_against_oracle(ev, ua, ia, users, g_train, g_held, Ks, is_val):
    """Full mode == the oracle on the kernel's scores (AUC to 1e-12, NaN in the same places) and == part mode's ranking."""
    from mmssl_b200.evaluate import Evaluator
    out = ev.rank(torch.from_numpy(ua).cuda(), torch.from_numpy(ia).cuda(), users, is_val, want_scores=True)
    torch.cuda.synchronize()
    s_gpu = out["scores"].cpu().numpy()
    ref = FO.evaluate(ua, ia, users, g_train[0], g_train[1], g_held[0], g_held[1], Ks, rating=s_gpu)
    auc = out["auc"].cpu().numpy()
    _same_nan(auc, ref["auc_per_user"])
    np.testing.assert_allclose(auc, ref["auc_per_user"], rtol=0, atol=1e-12)
    assert np.array_equal(out["ranked"].cpu().numpy().astype(np.int64), ref["ranked"])
    np.testing.assert_allclose(out["per_user"].cpu().numpy(), ref["per_user"], rtol=0, atol=1e-12)
    # part mode on the same inputs: ranked, hits and per_user bitwise equal
    part = Evaluator(ev._train_rows, ev._held_rows[False], ev._held_rows[True], ev.n_users, ev.n_items, ev.Ks)
    po = part.rank(torch.from_numpy(ua).cuda(), torch.from_numpy(ia).cuda(), users, is_val)
    for k in ("ranked", "ranked_scores", "hits", "per_user", "result"):
        assert torch.equal(po[k].cpu(), out[k].cpu()), k
    # a second full-mode run is bitwise equal
    again = ev.rank(torch.from_numpy(ua).cuda(), torch.from_numpy(ia).cuda(), users, is_val)
    assert np.array_equal(again["auc"].cpu().numpy().view(np.int64), auc.view(np.int64))
    # test_torch: 'auc' is the mean of rank()["auc"]
    res = ev.test_torch(torch.from_numpy(ua).cuda(), torch.from_numpy(ia).cuda(), list(users), is_val)
    mean = float(np.mean(auc)) if len(auc) else 0.
    assert (np.isnan(res["auc"]) and np.isnan(mean)) or abs(res["auc"] - mean) <= 1e-12
    assert (np.isnan(res["auc"]) and np.isnan(ref["auc"])) or abs(res["auc"] - ref["auc"]) <= 1e-12
    return out, s_gpu


class _Ev:
    """Evaluator in full mode that remembers its rows, so the part-mode twin can be built from the same input."""

    def __new__(cls, train, test, val, U, I, Ks):
        from mmssl_b200.evaluate import Evaluator
        ev = Evaluator(train, test, val, U, I, Ks, test_flag="full")
        ev._train_rows, ev._held_rows = train, {False: test, True: val}
        return ev


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("split", ["test", "val"])
def test_eval_full_matches_reference_golden(case, split):
    g = np.load(os.path.join(GOLD, case + ".npz"))
    Ks = [int(k) for k in g["Ks"]]
    U, I = g["ua"].shape[0], g["ia"].shape[0]
    ev = _Ev(_rows(g["train_indptr"], g["train_indices"]), _rows(g["test_indptr"], g["test_indices"]),
             _rows(g["val_indptr"], g["val_indices"]), U, I, Ks)
    users = g[f"{split}_users"]
    held = (g[f"{split}_indptr"], g[f"{split}_indices"])
    out, _ = check_against_oracle(ev, g["ua"], g["ia"], users, (g["train_indptr"], g["train_indices"]), held, Ks, split == "val")
    auc, want = out["auc"].cpu().numpy(), g[f"{split}_auc_per_user"]
    _same_nan(auc, want)
    if case in ("eval_full_ties", "eval_full_edges"):
        # quantised embeddings: every score is exact in fp32 whatever the summation order, so the reference's own AUC
        np.testing.assert_allclose(auc, want, rtol=0, atol=1e-12)
    else:
        # fp32 scores summed in another order than the reference's matmul can differ in the last bit, which can reorder
        # at most the one pair whose two scores are that close: per user |delta| <= 1 / (|P| |N|) (+ fp64 rounding)
        tp, ti, hp, hi = g["train_indptr"], g["train_indices"], held[0], held[1]
        for k, u in enumerate(users):
            if np.isnan(want[k]):
                continue
            cand = np.setdiff1d(np.arange(I), ti[tp[u]:tp[u + 1]])
            P = int(np.isin(cand, hi[hp[u]:hp[u + 1]]).sum())
            assert abs(auc[k] - want[k]) <= 1.0 / (P * (len(cand) - P)) + 1e-12, (k, auc[k], want[k])


def test_eval_full_random_tie_heavy_cases():
    """Small-integer embeddings (many exact ties between positives and negatives), positives counts on both sides of the
    kernel's 128-key shared-memory stage, duplicate held ids, empty and near-full training rows."""
    rng = np.random.default_rng(321)
    for case in range(6):
        U, I = int(rng.integers(1, 20)), int(rng.integers(2, 900))
        d = int(rng.choice([4, 16, 64]))
        Ks = sorted(set(int(k) for k in rng.integers(1, 65, int(rng.integers(1, 4)))))
        ua = rng.integers(-2, 3, (U, d)).astype(np.float32)
        ia = rng.integers(-2, 3, (I, d)).astype(np.float32)
        train = {u: sorted(rng.choice(I, size=int(rng.integers(0, I)), replace=False).tolist()) for u in range(U)}
        held = {u: rng.choice(I, size=int(rng.choice([rng.integers(1, 8), rng.integers(100, 400)])), replace=True).tolist()
                for u in range(U)}
        train = {u: v for u, v in train.items() if v}
        ev = _Ev(train, held, {}, U, I, Ks)
        check_against_oracle(ev, ua, ia, rng.permutation(U).astype(np.int64), _csr(train, U), _csr(held, U), Ks, False)


def test_eval_full_baby_size_heavy_user():
    """Baby-sized tables (19445 x 7050, d=64), every user evaluated, one user with 3000 positives."""
    from mmssl_b200.synthetic import CONFIGS, make_bipartite
    U, I, nnz, d, *_ = CONFIGS["baby"]
    tr = make_bipartite(U, I, nnz, seed=3).tocsr()
    tr.sort_indices()
    rng = np.random.default_rng(1)
    held = {u: rng.choice(I, size=int(rng.integers(1, 6)), replace=False).tolist() for u in range(U)}
    held[77] = rng.choice(I, size=3000, replace=False).tolist()
    ua = rng.standard_normal((U, d)).astype(np.float32)
    ia = rng.standard_normal((I, d)).astype(np.float32)
    train_rows = {u: tr.indices[tr.indptr[u]:tr.indptr[u + 1]].tolist() for u in range(U) if tr.indptr[u + 1] > tr.indptr[u]}
    ev = _Ev(train_rows, held, {}, U, I, [10, 20, 50])
    users = np.arange(U, dtype=np.int64)
    check_against_oracle(ev, ua, ia, users, (tr.indptr.astype(np.int64), tr.indices.astype(np.int64)), _csr(held, U),
                         [10, 20, 50], False)


def run_trainer_full(device="cuda"):
    """A Trainer life cycle with test_flag='full': test() reports the AUC an Evaluator computes on the same embeddings."""
    from mmssl_b200.dataset import ReferenceDataset
    from mmssl_b200.evaluate import Evaluator
    from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed
    ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
    args = TrainerArgs(dataset="dataset_small", epoch=1, batch_size=16, verbose=1, early_stopping_patience=1, m_topk_rate=0.05,
                       Ks="[2, 5, 10]", seed=5, test_flag="full")
    set_seed(args.seed)
    tr = Trainer(ds, args, device=device, log=None)
    _, test_ret = tr.train()
    assert test_ret is not None and isinstance(test_ret["auc"], float)
    users = sorted(ds.test_set)
    ret = tr.test(users, is_val=False)
    hs = tr.step.hs
    outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, None, want_sumsq=False)
    ev = Evaluator(ds.train_items, ds.test_set, ds.val_set, tr.n_users, tr.n_items, tr.Ks, device=device, test_flag="full")
    want = ev.test_torch(outs[0], outs[1], users, False)
    assert np.array_equal(np.float64(ret["auc"]), np.float64(want["auc"]), equal_nan=True)
    for k in ("precision", "recall", "ndcg", "hit_ratio"):
        assert np.array_equal(ret[k], want[k])
    with pytest.raises(ValueError):
        Evaluator(ds.train_items, ds.test_set, ds.val_set, tr.n_users, tr.n_items, tr.Ks, device=device, test_flag="fast")


def test_trainer_full_mode_auc():
    run_trainer_full()
