"""The full-mode oracle (tests/eval_full_oracle.py) against the golden vectors minted from the reference run with
--test_flag full, and against sklearn's roc_auc_score itself."""
import os
import warnings

import numpy as np
import pytest

from tests import eval_full_oracle as FO

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["eval_full_random", "eval_full_ties", "eval_full_short", "eval_full_edges"]


def _same(a, b, atol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    np.testing.assert_allclose(a[~np.isnan(a)], b[~np.isnan(b)], rtol=0, atol=atol)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("split", ["test", "val"])
def test_auc_user_matches_reference_golden(case, split):
    g = np.load(os.path.join(GOLD, case + ".npz"))
    tp, ti = g["train_indptr"], g["train_indices"]
    hp, hi = g[f"{split}_indptr"], g[f"{split}_indices"]
    users = g[f"{split}_users"]
    rating = g[f"{split}_rating"]
    got = [FO.auc_user(rating[k], ti[tp[u]:tp[u + 1]], hi[hp[u]:hp[u + 1]]) for k, u in enumerate(users)]
    _same(got, g[f"{split}_auc_per_user"], 1e-12)
    out = FO.evaluate(g["ua"], g["ia"], users, tp, ti, hp, hi, [int(k) for k in g["Ks"]], rating=rating)
    _same(out["auc_per_user"], g[f"{split}_auc_per_user"], 1e-12)
    _same(out["auc"], g[f"{split}_result_auc"], 1e-12)
    np.testing.assert_allclose(out["result"], g[f"{split}_result"], rtol=0, atol=1e-12)


def test_edges_golden_covers_every_branch():
    g = np.load(os.path.join(GOLD, "eval_full_edges.npz"))
    a = g["test_auc_per_user"]
    assert np.isnan(a).sum() >= 2 and np.isfinite(a).sum() >= 10
    lens = np.diff(g["test_indptr"])[g["test_users"]]
    assert lens.max() >= 1500 and (lens == 128).any() and (lens == 129).any()
    r = g["test_rating"]
    assert len(np.unique(r)) < r.size // 100                          # quantised: many exact ties


def _sk(labels, scores):
    from sklearn.metrics import roc_auc_score
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return float(roc_auc_score(y_true=labels, y_score=scores))
    except Exception:                                                 # metrics.py:97-99
        return 0.


def _check_vs_sklearn(rating, train, held):
    cand = np.setdiff1d(np.arange(rating.shape[0]), train)
    labels = np.isin(cand, held).astype(int)
    want = _sk(labels, rating[cand])
    got = FO.auc_user(rating, train, held)
    _same([got], [want], 1e-12)


def test_auc_user_matches_sklearn():
    pytest.importorskip("sklearn")
    rng = np.random.default_rng(7)
    for case in range(60):
        I = int(rng.integers(1, 400))
        if case % 2:
            rating = rng.integers(-3, 4, I).astype(np.float32)            # tie-heavy
        else:
            rating = rng.standard_normal(I).astype(np.float32)
        train = rng.choice(I, size=int(rng.integers(0, I + 1)), replace=False)
        held = rng.choice(I, size=int(rng.integers(0, I + 1)), replace=True)      # duplicates, overlaps with train
        _check_vs_sklearn(rating, train, held)


def test_auc_user_one_class_and_non_finite():
    pytest.importorskip("sklearn")
    r = np.array([0.5, -1.0, 2.0, 0.0, 3.0], np.float32)
    _check_vs_sklearn(r, np.array([0, 1]), np.array([0, 1]))           # no positive -> NaN
    assert np.isnan(FO.auc_user(r, np.array([0, 1]), np.array([0, 1])))
    _check_vs_sklearn(r, np.array([0, 1]), np.array([2, 3, 4]))        # no negative -> NaN
    _check_vs_sklearn(r, np.arange(5), np.array([2]))                  # no candidate -> 0
    assert FO.auc_user(r, np.arange(5), np.array([2])) == 0.
    for bad in (np.nan, np.inf, -np.inf):
        rb = r.copy()
        rb[3] = bad
        _check_vs_sklearn(rb, np.array([0]), np.array([2]))            # non-finite candidate -> 0
        assert FO.auc_user(rb, np.array([0]), np.array([2])) == 0.
        assert FO.auc_user(rb, np.array([3]), np.array([2])) == FO.auc_user(r, np.array([3]), np.array([2]))   # a training item's score is not looked at
