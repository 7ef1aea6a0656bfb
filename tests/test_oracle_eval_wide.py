"""oracle/eval_oracle.py against the golden vectors minted from the unmodified reference with wide cut-off lists
(tests/golden/make_golden_eval_wide.py): 12 or 13 cut-offs, unsorted, with a duplicate, K in 1..1000, max(Ks) > n_items,
and one --test_flag full case (whose AUC the full-mode oracle reproduces)."""
import json
import os

import numpy as np
import pytest

from oracle import eval_oracle as EO
from tests import eval_full_oracle as FO

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["eval_wide_random", "eval_wide_ties", "eval_wide_short", "eval_wide_full"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("split", ["test", "val"])
def test_eval_oracle_matches_reference_wide(case, split):
    g = np.load(os.path.join(GOLD, case + ".npz"))
    Ks = [int(k) for k in g["Ks"]]
    rating = g[f"{split}_rating"] if f"{split}_rating" in g else None
    out = EO.evaluate(g["ua"], g["ia"], g[f"{split}_users"], g["train_indptr"], g["train_indices"], g[f"{split}_indptr"],
                      g[f"{split}_indices"], Ks, rating=rating)
    assert out["ranked"].shape == g[f"{split}_ranked"].shape == (len(g[f"{split}_users"]), max(Ks))
    assert np.array_equal(out["ranked"], g[f"{split}_ranked"])          # incl. the tie order
    assert np.array_equal(out["hits"], g[f"{split}_hits"])
    np.testing.assert_allclose(out["per_user"], g[f"{split}_per_user"], rtol=0, atol=1e-15)
    np.testing.assert_allclose(out["result"], g[f"{split}_result"], rtol=0, atol=1e-14)
    if rating is not None:
        fo = FO.evaluate(g["ua"], g["ia"], g[f"{split}_users"], g["train_indptr"], g["train_indices"], g[f"{split}_indptr"],
                         g[f"{split}_indices"], Ks, rating=rating)
        a, want = fo["auc_per_user"], g[f"{split}_auc_per_user"]
        assert np.array_equal(np.isnan(a), np.isnan(want))
        np.testing.assert_allclose(a[~np.isnan(a)], want[~np.isnan(want)], rtol=0, atol=1e-12)


def test_wide_goldens_cover_the_cases():
    """The cut-off lists, the tie density and the short list the goldens were minted for."""
    g = np.load(os.path.join(GOLD, "eval_wide_random.npz"))
    Ks = [int(k) for k in g["Ks"]]
    assert len(Ks) >= 12 and {64, 65, 100, 128, 1000} <= set(Ks) and len(set(Ks)) < len(Ks) and Ks != sorted(Ks)
    t = np.load(os.path.join(GOLD, "eval_wide_ties.npz"))
    r = EO.scores(t["ua"], t["ia"], t["test_users"])
    assert len(np.unique(r)) < r.size // 100
    s = np.load(os.path.join(GOLD, "eval_wide_short.npz"))
    assert max(int(k) for k in s["Ks"]) > s["ia"].shape[0] and (s["test_ranked"] == -1).any()
    f = np.load(os.path.join(GOLD, "eval_wide_full.npz"))
    assert json.loads(str(f["cfg"]))["test_flag"] == "full" and max(int(k) for k in f["Ks"]) > 64


def test_ndcg_ideal_uses_the_whole_retrieved_list():
    """metrics.py:68-70: the ideal DCG at K is built from the hits of the whole list of length max(Ks), so adding a
    cut-off of 100 changes ndcg@10 when a hit sits at ranks 10..99 -- the reference's quirk, kept."""
    hits = np.zeros(100, np.int64)
    hits[[3, 40]] = 1
    short = EO.user_metrics(hits[:50], 2, [10, 20, 50])
    wide = EO.user_metrics(hits, 2, [10, 20, 50, 100])
    assert np.array_equal(short[:2], wide[:2, :3]) and np.array_equal(short[3], wide[3, :3])
    assert wide[2, 0] == short[2, 0]                                  # both lists hold the hit at 40
    only = EO.user_metrics(hits[:20], 2, [10, 20])
    assert only[2, 0] != wide[2, 0]                                   # the list of 20 does not
