"""CPU oracle for full-mode evaluation (``--test_flag full``).  TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Restates in numpy what the reference adds in that mode (citations relative to MMSSL/ of the reference repository):
``test_one_user`` calls ``ranklist_by_sorted`` instead of ``ranklist_by_heapq`` (utility/batch_test.py:104-107), whose
``get_auc`` (:38-51) hands the labels of every non-training item and their scores to ``metrics.auc`` ->
``sklearn.metrics.roc_auc_score`` (utility/metrics.py:95-100); ``test_torch`` averages it over the users (:165).  The
top-K list, hits and the four metrics are those of part mode (``oracle/eval_oracle.py``).

Quirks kept on purpose (sklearn 1.9, as the reference runs with it):
  * held-out items that are also training items are in neither class; duplicate ids count once;
  * one class only (no positive, or every candidate a positive): roc_auc_score warns and returns NaN, metrics.auc
    passes it on, so the reference's mean AUC is NaN as soon as one such user is evaluated;
  * a NaN / inf candidate score, or no candidate at all: roc_auc_score raises, metrics.auc returns 0.

PARITY PIN: ``tests/golden/eval_full_*.npz`` minted by ``tests/golden/make_golden_eval_full.py`` from the unmodified
reference; ``tests/test_oracle_eval_full.py`` checks this file against them and against sklearn.
"""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np

from oracle import eval_oracle as EO


def auc_user(rating: np.ndarray, train: np.ndarray, held: np.ndarray) -> float:
    """roc_auc_score(labels, scores) over the items of ``rating`` [I] that are not in ``train``, labels = membership in
    ``held``: (#pairs ordered right + 1/2 #tied pairs) / (|P| |N|), from exact integer counts."""
    rating = np.asarray(rating, np.float32)
    n_items = rating.shape[0]

    def inside(a):
        a = np.asarray(a, np.int64)
        return a[(a >= 0) & (a < n_items)]
    cand = np.ones(n_items, bool)
    cand[inside(train)] = False
    if not cand.any():
        return 0.0
    if not np.isfinite(rating[cand]).all():
        return 0.0
    pos = np.zeros(n_items, bool)
    pos[inside(held)] = True
    pos &= cand
    P = int(pos.sum())
    N = int(cand.sum()) - P
    if P == 0 or N == 0:
        return float("nan")
    sp = np.sort(rating[pos])
    sn = rating[cand & ~pos]
    lt = np.searchsorted(sp, sn, side="left").astype(np.int64)        # #{s_p < s_n}
    le = np.searchsorted(sp, sn, side="right").astype(np.int64)       # #{s_p <= s_n}
    num = int((2 * (P - le) + (le - lt)).sum())
    return num / (2.0 * P * N)


def evaluate(ua: np.ndarray, ia: np.ndarray, users: Sequence[int], train_indptr: np.ndarray, train_indices: np.ndarray,
             held_indptr: np.ndarray, held_indices: np.ndarray, Ks: Sequence[int],
             rating: np.ndarray | None = None) -> Dict[str, np.ndarray]:
    """``eval_oracle.evaluate`` plus auc_per_user [n] and auc (their mean accumulated in user order, batch_test.py:165)."""
    users = np.asarray(users, np.int64)
    if rating is None:
        rating = EO.scores(ua, ia, users)
    out = EO.evaluate(ua, ia, users, train_indptr, train_indices, held_indptr, held_indices, Ks, rating=rating)
    n = len(users)
    auc = np.array([auc_user(rating[k], train_indices[train_indptr[u]:train_indptr[u + 1]],
                             held_indices[held_indptr[u]:held_indptr[u + 1]]) for k, u in enumerate(users)])
    mean = 0.
    for k in range(n):
        mean += auc[k] / n
    out.update(auc_per_user=auc, auc=mean)
    return out
