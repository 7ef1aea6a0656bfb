#!/usr/bin/env python
"""Mint golden vectors for evaluation with wide cut-off lists (more than 8 cut-offs, K > 64, K > n_items) from the
UNMODIFIED reference (utility/batch_test.py + metrics.py of the checkout named by $MMSSL_REFERENCE), run on CPU.

    python tests/golden/make_golden_eval_wide.py        # writes tests/golden/eval_wide_*.npz

Datasets and embeddings are made by make_golden_eval.py's generator (whose eval_*.npz stay as they are).  Per split the
file holds what make_golden_eval.py stores (result, per_user, hits, ranked -- ranked / hits [n, max(Ks)], -1 padded); the
``--test_flag full`` case also holds ``{split}_rating``, ``{split}_auc_per_user`` and ``{split}_result_auc`` like
make_golden_eval_full.py.  ``test_one_user`` -> ``ranklist_by_heapq`` / ``ranklist_by_sorted`` -> ``get_performance`` is
executed, not restated; with max(Ks) >= #candidates ``heapq.nlargest`` takes its stable ``sorted`` branch.
"""
import argparse
import heapq
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_eval as base  # noqa: E402

# 12 or 13 cut-offs, unsorted, with a duplicate, across 64 / 65, 100, 128 and 1000
WIDE = "[100, 10, 65, 1000, 20, 64, 5, 128, 50, 1, 200, 100]"
CASES = {
    # random fp32 embeddings; max(Ks) = 1000 < 1500 items: the heapq branch
    "eval_wide_random": dict(U=40, I=1500, d=16, seed=31, quant=0, ks=WIDE, flag="part"),
    # embeddings quantised to multiples of 1/4: many exactly equal scores -> tie order (lower item id first) matters
    "eval_wide_ties": dict(U=50, I=1200, d=8, seed=33, quant=4, ks="[65, 64, 1000, 128, 10, 20, 300, 5, 1, 2, 3, 100, 65]", flag="part"),
    # max(Ks) > n_items: every candidate is ranked (heapq.nlargest's sorted branch), the hit list is shorter than K
    "eval_wide_short": dict(U=30, I=90, d=8, seed=35, quant=0, ks="[5, 100, 64, 65, 128, 1000, 20, 10, 1, 2, 3, 90, 91]", flag="part"),
    # --test_flag full: ranklist_by_sorted + the per-user ROC-AUC, with wide Ks
    "eval_wide_full": dict(U=40, I=800, d=16, seed=37, quant=2, ks=WIDE, flag="full"),
}


def run_case(name):
    import importlib
    import torch

    c = CASES[name]
    tmp = tempfile.mkdtemp(prefix="mmssl_golden_eval_wide_")
    base.make_dataset(tmp, name, c["U"], c["I"], c["seed"])
    if not hasattr(np, "asfarray"):
        np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)
    sys.path.insert(0, base.REF)
    os.chdir(base.REF)
    sys.argv = ["main.py", "--dataset", name, "--data_path", tmp + "/", "--debug", "--Ks", c["ks"], "--test_flag", c["flag"]]
    bt = importlib.import_module("utility.batch_test")
    assert bt.args.test_flag == c["flag"]
    dg = bt.data_generator
    U, I = dg.n_users, dg.n_items
    assert (U, I) == (c["U"], c["I"]), (U, I)
    Ks = bt.Ks
    rng = np.random.default_rng(c["seed"] + 100)
    ua = rng.standard_normal((U, c["d"])).astype(np.float32)
    ia = rng.standard_normal((I, c["d"])).astype(np.float32)
    if c["quant"]:
        ua = np.round(ua * c["quant"] / 2) / c["quant"]
        ia = np.round(ia * c["quant"] / 2) / c["quant"]
    ua_t, ia_t = torch.from_numpy(ua), torch.from_numpy(ia)
    full = c["flag"] == "full"

    out = dict(ua=ua, ia=ia, Ks=np.array(Ks, np.int64))
    out["train_indptr"], out["train_indices"] = base.ragged(dg.train_items, U)
    for split, is_val in (("test", False), ("val", True)):
        held = dg.val_set if is_val else dg.test_set
        users = list(held.keys())
        out[f"{split}_indptr"], out[f"{split}_indices"] = base.ragged(held, U)
        out[f"{split}_users"] = np.array(users, np.int64)
        res = bt.test_torch(ua_t, ia_t, users, is_val)                    # the reference's aggregate
        out[f"{split}_result"] = np.stack([res[k] for k in ("precision", "recall", "ndcg", "hit_ratio")])
        kmax = max(Ks)
        per_user = np.zeros((len(users), 4, len(Ks)))
        hits = -np.ones((len(users), kmax), np.int64)
        ranked = -np.ones((len(users), kmax), np.int64)
        rating_all = np.zeros((len(users), I), np.float32)
        auc = np.zeros(len(users))
        for n, u in enumerate(users):
            rating = torch.matmul(ua_t[[u]], ia_t.t())[0].numpy()        # the row test_torch hands to test_one_user
            rating_all[n] = rating
            p = bt.test_one_user((rating, u, is_val))
            per_user[n] = np.stack([p[k] for k in ("precision", "recall", "ndcg", "hit_ratio")])
            auc[n] = p["auc"]
            test_items = list(set(range(I)) - set(dg.train_items.get(u, [])))
            rank_fn = bt.ranklist_by_sorted if full else bt.ranklist_by_heapq
            r, _ = rank_fn(held[u], test_items, rating, Ks)
            hits[n, :len(r)] = r
            score = {i: rating[i] for i in test_items}                    # same call as batch_test.py:26-27
            top = heapq.nlargest(kmax, score, key=score.get)
            ranked[n, :len(top)] = top
        out[f"{split}_per_user"], out[f"{split}_hits"], out[f"{split}_ranked"] = per_user, hits, ranked
        if full:
            out[f"{split}_result_auc"] = np.float64(res["auc"])
            out[f"{split}_rating"], out[f"{split}_auc_per_user"] = rating_all, auc
    out["cfg"] = np.array(json.dumps(dict(U=U, I=I, d=c["d"], Ks=Ks, test_flag=bt.args.test_flag, numpy=np.__version__,
                                          torch=torch.__version__)))
    dst = os.path.join(HERE, name + ".npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst) // 1024, "KiB; recall@Ks", out["test_result"][1])


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    a, _ = ap.parse_known_args()
    if a.case:
        run_case(a.case)
    else:
        for n in CASES:
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--case", n])
