#!/usr/bin/env python
"""Mint golden vectors from the UNMODIFIED reference (a checkout of HKUDS/MMSSL named by $MMSSL_REFERENCE), run on CPU.

Runs only where that checkout exists; the tests read the stored vectors.  One sub-process per case
because the reference parses its CLI flags at import time in four modules.

    python tests/golden/make_golden.py            # writes tests/golden/case_*.npz

Import recipe = SURVEY.md appendix C: stub the import-only deps (dgl, visdom), make `.cuda()` an
identity, `--debug` to disable the hard-coded log path, chdir into MMSSL/ so `utility.*` resolves.
No reference source is copied; the reference modules are imported and executed as they are.
"""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
import types

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MMSSL_REFERENCE", "MMSSL")      # the directory holding the reference's main.py

CASES = {
    # name: (n_users, n_items, dv, dt, batch, weight_size, graph mode, train mode, seed)
    "case_eval_alias_k2": dict(U=257, I=131, dv=96, dt=40, B=64, ws="[64,64]", modal="alias", train=False, seed=2022),
    "case_train_rand_k3": dict(U=203, I=150, dv=72, dt=24, B=96, ws="[64,64,64]", modal="random", train=True, seed=7),
    "case_train_empty_k2": dict(U=180, I=97, dv=40, dt=56, B=50, ws="[64,64]", modal="empty", train=True, seed=11),
}


def make_dataset(root, name, U, I, dv, dt, seed):
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for u in range(U):
        deg = int(np.clip(rng.lognormal(1.2, 0.8), 1, I // 2))
        its = rng.choice(I, size=deg, replace=False, p=None)
        rows += [u] * deg
        cols += its.tolist()
    # make sure the last item id appears (n_items is inferred from the json files)
    rows.append(0)
    cols.append(I - 1)
    mat = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(U, I))
    mat.data[:] = 1.0  # duplicates collapse to 1
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    train = {str(u): mat.indices[mat.indptr[u]:mat.indptr[u + 1]].tolist() for u in range(U)}
    held = {str(u): [int(rng.integers(0, I))] for u in range(0, U, 3)}
    for fn, obj in (("train.json", train), ("val.json", held), ("test.json", held)):
        with open(os.path.join(d, fn), "w") as f:
            json.dump(obj, f)
    with open(os.path.join(d, "train_mat"), "wb") as f:
        pickle.dump(mat, f)
    np.save(os.path.join(d, "image_feat.npy"), rng.standard_normal((I, dv)).astype(np.float32))
    np.save(os.path.join(d, "text_feat.npy"), rng.standard_normal((I, dt)).astype(np.float32))
    return mat


def run_case(name):
    import importlib
    import torch
    import torch.nn as nn

    c = CASES[name]
    tmp = tempfile.mkdtemp(prefix="mmssl_golden_")
    make_dataset(tmp, name, c["U"], c["I"], c["dv"], c["dt"], c["seed"])

    sys.path.insert(0, REF)
    os.chdir(REF)
    sys.argv = ["main.py", "--dataset", name, "--data_path", tmp + "/", "--debug",
                "--batch_size", str(c["B"]), "--weight_size", c["ws"]]
    for m in ("dgl", "visdom"):
        sys.modules[m] = types.ModuleType(m)
    torch.Tensor.cuda = lambda s, *a, **k: s
    nn.Module.cuda = lambda s, *a, **k: s
    torch.cuda.manual_seed_all = lambda s: None
    torch.set_num_threads(4)

    main = importlib.import_module("main")
    main.set_seed(c["seed"])
    tr = main.Trainer({})
    model = tr.model
    U, I = tr.n_users, tr.n_items
    rng = np.random.default_rng(c["seed"] + 1)

    # --- modality graphs ---------------------------------------------------------------
    def rand_graph(shape, nnz):
        r = rng.integers(0, shape[0], nnz)
        q = rng.integers(0, shape[1], nnz)
        m = sp.csr_matrix((np.ones(nnz), (r, q)), shape=shape)  # duplicates are summed -> values > 1
        return tr.sparse_mx_to_torch_sparse_tensor(tr.csr_norm(m, mean_flag=True))

    if c["modal"] == "alias":
        graphs = [tr.ui_graph, tr.iu_graph, tr.ui_graph, tr.iu_graph, tr.ui_graph, tr.iu_graph]
    elif c["modal"] == "random":
        g_img = rand_graph((U, I), 700)
        g_txt = rand_graph((U, I), 500)
        graphs = [tr.ui_graph, tr.iu_graph, g_img, rand_graph((I, U), 650), g_txt, rand_graph((I, U), 300)]
    else:
        empty_ui = tr.sparse_mx_to_torch_sparse_tensor(tr.csr_norm(sp.csr_matrix((U, I)), mean_flag=True))
        empty_iu = tr.sparse_mx_to_torch_sparse_tensor(tr.csr_norm(sp.csr_matrix((I, U)), mean_flag=True))
        graphs = [tr.ui_graph, tr.iu_graph, empty_ui, empty_iu, empty_ui, empty_iu]

    # --- dropout: inject fixed masks through the module attribute (reference code untouched) ---
    d = main.args.embed_size
    p = main.args.drop_rate
    masks = [(torch.from_numpy(rng.random((I, d))) >= p).float() / (1 - p) for _ in range(2)]

    class InjectedDropout(nn.Module):
        def __init__(self):
            super().__init__()
            self.calls = 0

        def forward(self, x):
            if not self.training:
                return x
            m = masks[self.calls % 2]
            self.calls += 1
            return x * m

    model.dropout = InjectedDropout()
    model.train() if c["train"] else model.eval()

    users, pos, neg = main.data_generator.sample()
    users = [int(u) for u in users]; pos = [int(x) for x in pos]; neg = [int(x) for x in neg]

    outs = model(*graphs)
    mf, emb, reg = tr.bpr_loss(outs[0][users], outs[1][pos], outs[1][neg])
    fr = tr.feat_reg_loss_calculation(outs[2], outs[3], outs[4], outs[5])
    cl1 = tr.batched_contrastive_loss(outs[8][users], outs[6][users])
    cl2 = tr.batched_contrastive_loss(outs[9][users], outs[6][users])
    cl_small_block = tr.batched_contrastive_loss(outs[8][users], outs[6][users], batch_size=16)
    total = mf + emb + reg + fr + main.args.cl_rate * (cl1 + cl2)
    for q in model.parameters():
        q.grad = None
    total.backward()

    def coo(t):
        t = t.coalesce() if not t.is_coalesced() and t._nnz() == 0 else t
        return t._indices().numpy().astype(np.int64), t._values().detach().numpy().astype(np.float32)

    out = {}
    for k, g in zip(("ui", "iu", "img_ui", "img_iu", "txt_ui", "txt_iu"), graphs):
        idx, val = coo(g)
        out[f"g_{k}_idx"], out[f"g_{k}_val"] = idx, val
        out[f"g_{k}_shape"] = np.array(g.shape, np.int64)
    raw = tr.ui_graph_raw.tocoo()
    out["train_rows"], out["train_cols"] = raw.row.astype(np.int64), raw.col.astype(np.int64)
    out["image_feats"] = model.image_feats.numpy()
    out["text_feats"] = model.text_feats.numpy()
    out["mask0"], out["mask1"] = masks[0].numpy(), masks[1].numpy()
    out["users"], out["pos"], out["neg"] = np.array(users), np.array(pos), np.array(neg)
    live = ("image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias",
            "user_id_embedding.weight", "item_id_embedding.weight",
            "weight_dict.w_self_attention_cat", "weight_dict.w_q", "weight_dict.w_k")
    named = dict(model.named_parameters())
    for k in live:
        out["p/" + k] = named[k].detach().numpy().copy()
        if named[k].grad is not None:
            out["grad/" + k] = named[k].grad.numpy().copy()
    out["grad_is_none"] = np.array([k for k, v in named.items() if v.grad is None])
    for j, o in enumerate(outs):
        out[f"out{j}"] = o.detach().numpy()
    out["alias_0_6"] = np.array(outs[0] is outs[6])
    out["alias_1_7"] = np.array(outs[1] is outs[7])
    for k, v in (("mf", mf), ("emb", emb), ("feat_reg", fr), ("cl1", cl1), ("cl2", cl2),
                 ("cl_small_block", cl_small_block), ("total", total)):
        out["loss/" + k] = np.array(float(v), np.float64)
    out["cfg"] = np.array(json.dumps(dict(
        U=U, I=I, d=d, n_layers=len(eval(c["ws"])), B=c["B"], train=c["train"], modal=c["modal"],
        head_num=main.args.head_num, id_cat_rate=main.args.id_cat_rate, model_cat_rate=main.args.model_cat_rate,
        drop_rate=p, tau=main.args.tau, cl_rate=main.args.cl_rate, emb_decay=tr.decay,
        feat_reg_decay=main.args.feat_reg_decay, torch=torch.__version__)))
    dst = os.path.join(HERE, name + ".npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst) // 1024, "KiB; total loss", float(total))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    a, _ = ap.parse_known_args()
    if a.case:
        run_case(a.case)
    else:
        for n in CASES:
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--case", n])
