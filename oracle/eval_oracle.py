"""CPU oracle for the evaluation path (SURVEY.md section 8f row 3).  TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Only ``tests/`` may import this module; nothing under ``mmssl_b200/`` does.

Restates in numpy what the reference computes in ``Trainer.test`` (citations relative to
MMSSL/ of the reference repository):

  * dense scoring of a user batch against all items            utility/batch_test.py:147-154
  * per user: drop the training items, take the max(Ks) best   utility/batch_test.py:21-36, :83-107
    remaining items (``heapq.nlargest`` over a dict filled in ascending item order: equal scores
    keep the LOWER item id first), mark which of them are held-out positives
  * precision / recall / ndcg / hit ratio at every K           utility/batch_test.py:67-80, utility/metrics.py:9-19, :43-87
  * mean over the evaluated users                              utility/batch_test.py:159-164

Quirks kept on purpose:
  * ndcg's ideal DCG is the DCG of the *retrieved* hit list sorted descending (metrics.py:70), not of all positives:
    hits at ranks K..max(Ks) still count towards the ideal at K;
  * precision@K is the mean over the retrieved list cut at K, so with fewer than K rankable items the divisor shrinks
    (metrics.py:17-18);
  * recall divides by ``len(user_pos_test)`` -- held-out items that are also training items can never be retrieved
    but stay in the denominator;
  * 'auc' is 0 in the default ``test_flag == 'part'`` mode (batch_test.py:35).

PARITY PIN: ``tests/golden/eval_*.npz`` minted by ``tests/golden/make_golden_eval.py`` from the unmodified reference
(``test_torch``, ``test_one_user``, ``ranklist_by_heapq``); ``tests/test_oracle_golden.py`` checks this file against them.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import numpy as np


def scores(ua: np.ndarray, ia: np.ndarray, users: Sequence[int]) -> np.ndarray:
    """fp32 ``ua[users] @ ia.T`` (batch_test.py:150-152)."""
    return np.asarray(ua, np.float32)[np.asarray(users, np.int64)] @ np.asarray(ia, np.float32).T


def rank_user(rating: np.ndarray, train_items: np.ndarray, kmax: int) -> np.ndarray:
    """Ids of the ``kmax`` best non-training items, best first; ties -> lower id first (batch_test.py:21-27)."""
    n_items = rating.shape[0]
    keep = np.ones(n_items, bool)
    keep[np.asarray(train_items, np.int64)] = False
    cand = np.nonzero(keep)[0]                                   # ascending ids
    order = np.argsort(-rating[cand], kind="stable")             # stable: equal scores stay in ascending-id order
    return cand[order[:kmax]]


def user_metrics(hits: np.ndarray, n_pos: int, Ks: Sequence[int]) -> np.ndarray:
    """[4, len(Ks)] = precision, recall, ndcg, hit_ratio of one hit list (batch_test.py:67-80)."""
    r = np.asarray(hits, np.float64)
    out = np.zeros((4, len(Ks)))
    ideal = np.sort(r)[::-1]
    for j, K in enumerate(Ks):
        rk = r[:K]
        disc = 1.0 / np.log2(np.arange(2, rk.size + 2))
        out[0, j] = rk.mean() if rk.size else np.nan                                   # metrics.py:17-18
        out[1, j] = rk.sum() / n_pos if n_pos else 0.0                                 # metrics.py:78-83
        dcg_max = float((ideal[:K] * disc).sum()) if rk.size else 0.0                  # metrics.py:70
        out[2, j] = float((rk * disc).sum()) / dcg_max if dcg_max else 0.0             # metrics.py:71-73
        out[3, j] = 1.0 if rk.sum() > 0 else 0.0                                       # metrics.py:85-90
    return out


def evaluate(ua: np.ndarray, ia: np.ndarray, users: Sequence[int], train_indptr: np.ndarray, train_indices: np.ndarray,
             held_indptr: np.ndarray, held_indices: np.ndarray, Ks: Sequence[int],
             rating: np.ndarray | None = None) -> Dict[str, np.ndarray]:
    """Returns result [4, nK] (mean over users), per_user [n, 4, nK], ranked [n, kmax] (-1 padded), hits [n, kmax].
    ``rating`` (optional, [n, I]) replaces the fp32 matmul so a test can rank somebody else's scores exactly."""
    kmax = max(Ks)
    users = np.asarray(users, np.int64)
    if rating is None:
        rating = scores(ua, ia, users)
    n = len(users)
    per_user = np.zeros((n, 4, len(Ks)))
    ranked = -np.ones((n, kmax), np.int64)
    hits = -np.ones((n, kmax), np.int64)
    for k, u in enumerate(users):
        tr = train_indices[train_indptr[u]:train_indptr[u + 1]]
        pos = held_indices[held_indptr[u]:held_indptr[u + 1]]
        top = rank_user(rating[k], tr, kmax)
        h = np.isin(top, pos).astype(np.int64)
        ranked[k, :len(top)] = top
        hits[k, :len(top)] = h
        per_user[k] = user_metrics(h, len(pos), Ks)
    result = np.zeros((4, len(Ks)))
    for k in range(n):                                           # batch_test.py:159-163 accumulates re/n in user order
        result += per_user[k] / n
    return dict(result=result, per_user=per_user, ranked=ranked, hits=hits)
