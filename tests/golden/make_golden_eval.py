#!/usr/bin/env python
"""Mint golden vectors for the evaluation path (SURVEY section 8f row 3) from the UNMODIFIED reference
(utility/batch_test.py + metrics.py of the checkout named by $MMSSL_REFERENCE), run on CPU.

    python tests/golden/make_golden_eval.py        # writes tests/golden/eval_*.npz

The reference modules are imported and executed as they are (`test_torch`, `test_one_user`,
`ranklist_by_heapq`); nothing is copied.  Only shim: `np.asfarray` (removed in NumPy 2, used at
metrics.py:50,75).  One sub-process per case because batch_test.py parses the CLI and loads the
dataset at import time.
"""
import argparse
import heapq
import json
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MMSSL_REFERENCE", "MMSSL")      # the directory holding the reference's main.py

CASES = {
    # random fp32 embeddings: almost no exact ties
    "eval_random": dict(U=211, I=300, d=64, seed=5, quant=0, ks="[10, 20, 50]"),
    # embeddings quantised to multiples of 1/4: many exactly equal scores -> tie order (lower item id first) matters
    "eval_ties": dict(U=97, I=180, d=16, seed=9, quant=4, ks="[10, 20, 50]"),
    # fewer rankable items than max(Ks): the hit list is shorter than K
    "eval_short": dict(U=40, I=37, d=8, seed=13, quant=0, ks="[5, 20, 50]"),
}


def make_dataset(root, name, U, I, seed):
    rng = np.random.default_rng(seed)
    train, test, val = {}, {}, {}
    for u in range(U):
        deg = int(np.clip(rng.lognormal(1.2, 0.8), 1, max(1, I // 3)))
        its = rng.choice(I, size=deg, replace=False)
        train[str(u)] = [int(x) for x in its]                      # unsorted, like the real files
        if u % 4 != 3:                                              # every 4th user has no held-out items
            n_t = int(rng.integers(1, 9))
            cand = rng.choice(I, size=n_t, replace=False)
            if u % 7 == 0:                                          # some held-out items are ALSO training items
                cand[0] = its[0]
            test[str(u)] = [int(x) for x in cand]
        if u % 3 == 0:
            val[str(u)] = [int(x) for x in rng.choice(I, size=int(rng.integers(1, 4)), replace=False)]
    train["0"] = sorted(set(train["0"]) | {I - 1})                  # n_items is inferred from the json files
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    for fn, obj in (("train.json", train), ("val.json", val), ("test.json", test)):
        with open(os.path.join(d, fn), "w") as f:
            json.dump(obj, f)
    rows = [u for u in range(U) for _ in train[str(u)]]
    cols = [i for u in range(U) for i in train[str(u)]]
    mat = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(U, I))
    with open(os.path.join(d, "train_mat"), "wb") as f:
        pickle.dump(mat, f)


def ragged(dic, U):
    indptr = np.zeros(U + 1, np.int64)
    flat = []
    for u in range(U):
        its = dic.get(u, [])
        flat += list(its)
        indptr[u + 1] = len(flat)
    return indptr, np.array(flat, np.int64)


def run_case(name):
    import importlib
    import torch

    c = CASES[name]
    tmp = tempfile.mkdtemp(prefix="mmssl_golden_eval_")
    make_dataset(tmp, name, c["U"], c["I"], c["seed"])
    if not hasattr(np, "asfarray"):
        np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)
    sys.path.insert(0, REF)
    os.chdir(REF)
    sys.argv = ["main.py", "--dataset", name, "--data_path", tmp + "/", "--debug", "--Ks", c["ks"]]
    bt = importlib.import_module("utility.batch_test")
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

    out = dict(ua=ua, ia=ia, Ks=np.array(Ks, np.int64))
    out["train_indptr"], out["train_indices"] = ragged(dg.train_items, U)
    for split, is_val in (("test", False), ("val", True)):
        held = dg.val_set if is_val else dg.test_set
        users = list(held.keys())
        out[f"{split}_indptr"], out[f"{split}_indices"] = ragged(held, U)
        out[f"{split}_users"] = np.array(users, np.int64)
        res = bt.test_torch(ua_t, ia_t, users, is_val)                    # the reference's aggregate (Pool + heapq)
        out[f"{split}_result"] = np.stack([res[k] for k in ("precision", "recall", "ndcg", "hit_ratio")])
        kmax = max(Ks)
        per_user = np.zeros((len(users), 4, len(Ks)))
        hits = -np.ones((len(users), kmax), np.int64)
        ranked = -np.ones((len(users), kmax), np.int64)
        for n, u in enumerate(users):
            rating = torch.matmul(ua_t[[u]], ia_t.t())[0].numpy()        # the row test_torch hands to test_one_user
            p = bt.test_one_user((rating, u, is_val))
            per_user[n] = np.stack([p[k] for k in ("precision", "recall", "ndcg", "hit_ratio")])
            test_items = list(set(range(I)) - set(dg.train_items.get(u, [])))
            r, _ = bt.ranklist_by_heapq(held[u], test_items, rating, Ks)
            hits[n, :len(r)] = r
            score = {i: rating[i] for i in test_items}                    # same call as batch_test.py:26-27
            top = heapq.nlargest(kmax, score, key=score.get)
            ranked[n, :len(top)] = top
        out[f"{split}_per_user"], out[f"{split}_hits"], out[f"{split}_ranked"] = per_user, hits, ranked
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
