#!/usr/bin/env python
"""Mint golden vectors for full-mode evaluation (``--test_flag full``: per-user ROC-AUC over every non-training item) from
the UNMODIFIED reference (utility/batch_test.py + metrics.py of the checkout named by $MMSSL_REFERENCE), run on CPU.

    python tests/golden/make_golden_eval_full.py        # writes tests/golden/eval_full_*.npz

Same datasets and embeddings as make_golden_eval.py (whose eval_*.npz stay as they are), plus ``eval_full_edges``.
``test_one_user`` -> ``ranklist_by_sorted`` -> ``get_auc`` -> ``metrics.auc`` -> ``sklearn.metrics.roc_auc_score`` is
executed, not restated.  Per split the file holds, besides what make_golden_eval.py stores, ``{split}_rating`` (the score
row of every evaluated user, fp32), ``{split}_auc_per_user`` and ``{split}_result_auc`` (the reference's test_torch mean).
"""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_eval as base  # noqa: E402

CASES = {"eval_full_" + k[len("eval_"):]: v for k, v in base.CASES.items()}
# quantised embeddings (exact ties between positives and negatives), I ~ 3000 items and held-out rows that exercise
# every branch of the kernel: all training items (one class -> NaN), every non-training item (one class -> NaN),
# duplicate ids, and positives counts below, at and above the 128 the kernel sorts in shared memory (1600 of them)
CASES["eval_full_edges"] = dict(U=24, I=3001, d=16, seed=21, quant=2, ks="[10, 20, 50]", edges=True)


def make_edges_dataset(root, name, U, I, seed):
    rng = np.random.default_rng(seed)
    train, test, val = {}, {}, {}
    for u in range(U):
        deg = int(np.clip(rng.lognormal(2.0, 1.0), 1, 400))
        train[u] = sorted(int(x) for x in rng.choice(I - 1, size=deg, replace=False))
    train[0] = train[0] + [I - 1]                                   # n_items is inferred from the json files
    rest = lambda u: np.setdiff1d(np.arange(I), train[u])
    for u in range(U):
        test[u] = [int(x) for x in rng.choice(rest(u), size=int(rng.integers(1, 9)), replace=False)]
        if u % 3 == 0:
            val[u] = [int(x) for x in rng.choice(rest(u), size=int(rng.integers(1, 4)), replace=False)]
    test[1] = train[1][:5]                                          # only training items: no positive
    test[2] = [int(x) for x in rest(2)]                             # every candidate is a positive: no negative
    test[3] = [5, 5, 7, 7, 7, 100] + [int(x) for x in rng.choice(rest(3), size=4, replace=False)]
    test[4] = [int(x) for x in rng.choice(rest(4), size=1600, replace=False)] + train[4][:3]
    test[5] = [int(x) for x in rng.choice(rest(5), size=128, replace=False)]
    test[6] = [int(x) for x in rng.choice(rest(6), size=129, replace=False)]
    test[7] = [int(x) for x in rng.choice(rest(7), size=300, replace=False)]
    val[9] = [int(x) for x in rng.choice(rest(9), size=700, replace=False)]
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    for fn, obj in (("train.json", train), ("val.json", val), ("test.json", test)):
        with open(os.path.join(d, fn), "w") as f:
            json.dump({str(k): list(rng.permutation(v).tolist()) for k, v in obj.items()}, f)    # unsorted, like the real files
    rows = [u for u in range(U) for _ in train[u]]
    cols = [i for u in range(U) for i in train[u]]
    mat = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(U, I))
    with open(os.path.join(d, "train_mat"), "wb") as f:
        pickle.dump(mat, f)


def run_case(name):
    import importlib
    import torch

    c = CASES[name]
    tmp = tempfile.mkdtemp(prefix="mmssl_golden_eval_full_")
    (make_edges_dataset if c.get("edges") else base.make_dataset)(tmp, name, c["U"], c["I"], c["seed"])
    if not hasattr(np, "asfarray"):
        np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)
    sys.path.insert(0, base.REF)
    os.chdir(base.REF)
    sys.argv = ["main.py", "--dataset", name, "--data_path", tmp + "/", "--debug", "--Ks", c["ks"], "--test_flag", "full"]
    bt = importlib.import_module("utility.batch_test")
    assert bt.args.test_flag == "full"
    dg = bt.data_generator
    U, I = dg.n_users, dg.n_items
    assert (U, I) == (c["U"], c["I"]), (U, I)
    Ks = bt.Ks
    rng = np.random.default_rng(c["seed"] + 100)                     # the embeddings of make_golden_eval.py
    ua = rng.standard_normal((U, c["d"])).astype(np.float32)
    ia = rng.standard_normal((I, c["d"])).astype(np.float32)
    if c["quant"]:
        ua = np.round(ua * c["quant"] / 2) / c["quant"]
        ia = np.round(ia * c["quant"] / 2) / c["quant"]
    ua_t, ia_t = torch.from_numpy(ua), torch.from_numpy(ia)

    out = dict(ua=ua, ia=ia, Ks=np.array(Ks, np.int64))
    out["train_indptr"], out["train_indices"] = base.ragged(dg.train_items, U)
    for split, is_val in (("test", False), ("val", True)):
        held = dg.val_set if is_val else dg.test_set
        users = list(held.keys())
        out[f"{split}_indptr"], out[f"{split}_indices"] = base.ragged(held, U)
        out[f"{split}_users"] = np.array(users, np.int64)
        res = bt.test_torch(ua_t, ia_t, users, is_val)                    # the reference's aggregate (Pool + get_auc)
        out[f"{split}_result"] = np.stack([res[k] for k in ("precision", "recall", "ndcg", "hit_ratio")])
        out[f"{split}_result_auc"] = np.float64(res["auc"])
        rating = np.zeros((len(users), I), np.float32)
        auc = np.zeros(len(users))
        for n, u in enumerate(users):
            rating[n] = torch.matmul(ua_t[[u]], ia_t.t())[0].numpy()     # the row test_torch hands to test_one_user
            auc[n] = bt.test_one_user((rating[n], u, is_val))["auc"]
        out[f"{split}_rating"], out[f"{split}_auc_per_user"] = rating, auc
    out["cfg"] = np.array(json.dumps(dict(U=U, I=I, d=c["d"], Ks=Ks, test_flag=bt.args.test_flag, numpy=np.__version__,
                                          torch=torch.__version__, sklearn=importlib.import_module("sklearn").__version__)))
    dst = os.path.join(HERE, name + ".npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst) // 1024, "KiB; auc", out["test_result_auc"], out["val_result_auc"])


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    a, _ = ap.parse_known_args()
    if a.case:
        run_case(a.case)
    else:
        for n in CASES:
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--case", n])
