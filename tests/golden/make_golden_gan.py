#!/usr/bin/env python
"""Mint a golden TRACE of the reference's full training step (GAN side included, SURVEY section 8f row 2) by running
the UNMODIFIED `Trainer.train()` of the reference's main.py ($MMSSL_REFERENCE) for three steps on CPU and recording what flows
through it.  Runs only where that checkout exists.

    python tests/golden/make_golden_gan.py        # writes tests/golden/gan_trace.npz

Nothing of the reference is copied or edited: it is imported (recipe = make_golden.py / SURVEY appendix C) and observed
through hooks --
  * forward hooks on the Discriminator (inputs / outputs of its 4 calls per step),
  * instance-attribute wrappers around `u_sim_calculation`, `gradient_penalty`, `sparse_mx_to_torch_sparse_tensor`,
    `data_generator.sample`,
  * optimizer step pre/post hooks (gradients before, parameters after),
  * every random draw is recorded: `torch.rand` (gradient-penalty alpha), `Tensor.uniform_` (Gumbel noise) and the dropout
    masks (the nn.Dropout modules are swapped for mask-recording ones through the module attributes).
Three steps with T=1 cover the three states of the modality graphs: alias of ui/iu (step 0), rebuilt from the top-k ids
of step 0 (used by step 2), and empty (built at step 2).
"""
import importlib
import json
import os
import sys
import tempfile
import types
from collections import defaultdict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, make_dataset  # noqa: E402

CASE = dict(name="gan_trace", U=120, I=96, dv=24, dt=16, B=32, ws="[64,64]", seed=3, steps=3, m_topk_rate=0.05)


def main():
    import torch
    import torch.nn as nn

    c = CASE
    tmp = tempfile.mkdtemp(prefix="mmssl_golden_gan_")
    make_dataset(tmp, c["name"], c["U"], c["I"], c["dv"], c["dt"], c["seed"])
    sys.path.insert(0, REF)
    os.chdir(REF)
    sys.argv = ["main.py", "--dataset", c["name"], "--data_path", tmp + "/", "--debug", "--batch_size", str(c["B"]),
                "--weight_size", c["ws"], "--epoch", "1", "--m_topk_rate", str(c["m_topk_rate"])]
    for m in ("dgl", "visdom"):
        sys.modules[m] = types.ModuleType(m)
    torch.Tensor.cuda = lambda s, *a, **k: s
    nn.Module.cuda = lambda s, *a, **k: s
    torch.cuda.manual_seed_all = lambda s: None
    torch.set_num_threads(4)
    if not hasattr(np, "asfarray"):
        np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)

    M = importlib.import_module("main")
    M.set_seed(c["seed"])
    tr = M.Trainer({})
    args = M.args
    dg = M.data_generator
    dg.n_train = (c["steps"] - 1) * c["B"]                  # n_batch = n_train // batch_size + 1 (main.py:325)
    rng = np.random.default_rng(c["seed"] + 5)
    T = defaultdict(list)
    rec = {"on": False}

    def keep(key, t):
        T[key].append(t.detach().clone().numpy() if torch.is_tensor(t) else np.asarray(t))
        return t

    # ---- random draws ----
    class RecDropout(nn.Module):
        def __init__(self, p, key):
            super().__init__()
            self.p, self.key = p, key

        def forward(self, x):
            if not self.training:
                return x
            m = torch.from_numpy(((rng.random(tuple(x.shape)) >= self.p) / (1.0 - self.p)).astype(np.float32))
            keep(self.key, m)
            return x * m

    tr.model.dropout = RecDropout(args.drop_rate, "mask_model")
    assert isinstance(tr.D.net[3], nn.Dropout) and isinstance(tr.D.net[7], nn.Dropout)
    tr.D.net[3] = RecDropout(args.G_drop1, "mask_d1")
    tr.D.net[7] = RecDropout(args.G_drop2, "mask_d2")
    orig_rand, orig_uniform = torch.rand, torch.Tensor.uniform_
    torch.rand = lambda *a, **k: keep("alpha", orig_rand(*a, **k)) if rec["on"] else orig_rand(*a, **k)

    def rec_uniform(self, *a, **k):
        out = orig_uniform(self, *a, **k)
        if rec["on"]:
            keep("gumbel_u", out)
        return out
    torch.Tensor.uniform_ = rec_uniform

    # ---- observation points ----
    orig_sample = dg.sample

    def rec_sample():
        s = orig_sample()
        keep("sample", np.array([[int(v) for v in x] for x in s], np.int64))
        return s
    dg.sample = rec_sample
    tr.D.register_forward_hook(lambda mod, inp, out: (keep("D_in", inp[0]), keep("D_out", out), None)[2])
    o_usim, o_gp, o_sp = tr.u_sim_calculation, tr.gradient_penalty, tr.sparse_mx_to_torch_sparse_tensor
    tr.u_sim_calculation = lambda users, uf, itf: keep("u_sim", o_usim(users, uf, itf))
    tr.gradient_penalty = lambda D, xr, xf: keep("gp", o_gp(D, xr, xf))

    def rec_graph(mx):
        t = o_sp(mx)
        tc = t.coalesce()
        keep("graph_idx", tc.indices()); keep("graph_val", tc.values()); keep("graph_shape", np.array(t.shape))
        return t
    tr.sparse_mx_to_torch_sparse_tensor = rec_graph

    d_names = [k for k, _ in tr.D.named_parameters()]
    d_state_names = list(tr.D.state_dict().keys())
    live = ["image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias", "user_id_embedding.weight",
            "item_id_embedding.weight", "weight_dict.w_self_attention_cat"]
    named = dict(tr.model.named_parameters())

    def d_pre(opt, a, k):
        for n, p in tr.D.named_parameters():
            keep("Dgrad/" + n, p.grad)

    def d_post(opt, a, k):
        for n, v in tr.D.state_dict().items():
            keep("Dstate/" + n, v)

    def g_pre(opt, a, k):
        for n in live:
            keep("Ggrad/" + n, named[n].grad)

    def g_post(opt, a, k):
        for n in live:
            keep("Gparam/" + n, named[n])
    tr.optim_D.register_step_pre_hook(d_pre); tr.optim_D.register_step_post_hook(d_post)
    tr.optimizer_D.register_step_pre_hook(g_pre); tr.optimizer_D.register_step_post_hook(g_post)
    dummy = {k: np.ones(3) for k in ("recall", "precision", "ndcg", "hit_ratio")}
    tr.test = lambda users, is_val: dict(dummy, auc=0.)

    out = {}
    for n, v in tr.D.state_dict().items():
        out["D0/" + n] = v.detach().clone().numpy()
    for n in live + ["weight_dict.w_q", "weight_dict.w_k"]:
        out["G0/" + n] = named[n].detach().clone().numpy()
    raw = tr.ui_graph_raw.tocoo()
    out["train_rows"], out["train_cols"] = raw.row.astype(np.int64), raw.col.astype(np.int64)
    out["image_feats"], out["text_feats"] = tr.model.image_feats.numpy(), tr.model.text_feats.numpy()

    rec["on"] = True
    tr.train()
    rec["on"] = False

    for k, v in T.items():
        shapes = {x.shape for x in v}
        if len(shapes) == 1:
            out[k] = np.stack(v)
        else:                                  # ragged (graphs of different nnz): one entry per record
            out[k + "/n"] = np.array(len(v))
            for j, x in enumerate(v):
                out[f"{k}/{j}"] = x
    out["cfg"] = np.array(json.dumps(dict(
        U=c["U"], I=c["I"], d=args.embed_size, n_layers=2, B=c["B"], steps=c["steps"], drop_rate=args.drop_rate,
        G_drop1=args.G_drop1, G_drop2=args.G_drop2, gp_rate=args.gp_rate, G_rate=args.G_rate, D_lr=args.D_lr, lr=args.lr,
        log_log_scale=args.log_log_scale, real_data_tau=args.real_data_tau, ui_pre_scale=args.ui_pre_scale,
        m_topk_rate=args.m_topk_rate, T=args.T, cl_rate=args.cl_rate, tau=args.tau, emb_decay=tr.decay,
        feat_reg_decay=args.feat_reg_decay, head_num=args.head_num, id_cat_rate=args.id_cat_rate,
        model_cat_rate=args.model_cat_rate, d_param_names=d_names, d_state_names=d_state_names, torch=torch.__version__)))
    dst = os.path.join(HERE, c["name"] + ".npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst) // 1024, "KiB")
    for k in sorted(out):
        if "/" not in k or k.endswith("/n"):
            print("  ", k, getattr(out[k], "shape", None))


if __name__ == "__main__":
    main()
