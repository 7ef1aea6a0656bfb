"""CPU oracle for the MMSSL hot path.  TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  Nothing under ``mmssl_b200/`` does.

It restates, op by op and on stock CPU torch, the algorithm of the reference's per-step hot
path (citations are relative to MMSSL/ of the reference repository):

  * graph normalisation            main.py:89-112, :513-520
  * MMSSL.forward                  Models.py:139-220
  * bpr_loss                       main.py:499-511
  * sim / batched_contrastive_loss main.py:211-249
  * feat_reg_loss_calculation      main.py:252-257
  * hot-step loss assembly         main.py:420 (without the GAN term)
  * AdamW on the model parameters  main.py:76-80, :427-429

The arithmetic of the path lives in PyTorch (third party, README pins ">=1.13", the image has
2.11.0); so the oracle is a torch-CPU program and gradients come from torch autograd -- the same
engine the reference itself uses.

PARITY PIN: the reference ships no tests / golden vectors (SURVEY.md section 8c), so the pin is
the unmodified reference itself, imported in the build container by
``tests/golden/make_golden.py``; its outputs are committed under ``tests/golden/*.npz`` and
``tests/test_oracle_golden.py`` checks this oracle against them (forward, losses, gradients).

Two forwards are provided:
  ``forward_literal``  follows the reference expression by expression (including the
                       multi-head "attention" with all its reshapes) -- this is what the CPU
                       baseline times;
  ``forward_closed``   the algebraically reduced form of SURVEY.md appendix A, used to
                       document what the CUDA path computes.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# configuration (defaults: utility/parser.py:54-55,60,64,72-77,82,94)
# --------------------------------------------------------------------------------------
@dataclass
class HotPathConfig:
    embed_size: int = 64          # parser.py:55
    n_layers: int = 2             # len(weight_size), parser.py:82
    head_num: int = 4             # parser.py:77
    id_cat_rate: float = 0.36     # parser.py:75
    model_cat_rate: float = 0.55  # parser.py:73
    drop_rate: float = 0.2        # parser.py:72
    tau: float = 0.5              # parser.py:94
    cl_rate: float = 0.03         # parser.py:60
    emb_decay: float = 1e-5       # regs[0], parser.py:64 / main.py:51-52
    feat_reg_decay: float = 1e-5  # parser.py:29
    batch_size: int = 1024        # parser.py:54
    feat_layers: int = 1          # args.layers, parser.py:12 (loop is idempotent)
    lr: float = 5.5e-4            # parser.py:65
    weight_decay: float = 1e-2    # torch AdamW default (main.py:76-80 passes none)


# --------------------------------------------------------------------------------------
# graph normalisation  (main.py:89-103 with mean_flag=True, main.py:105-112)
# --------------------------------------------------------------------------------------
def csr_norm(mat: sp.spmatrix, mean_flag: bool = True) -> sp.spmatrix:
    """D_row^{-1/2} * A  (and * D_col^{-1/2} when mean_flag is False), +1e-8 inside the power."""
    rs = np.asarray(mat.sum(1))
    rs = np.power(rs + 1e-8, -0.5).ravel()
    rs[np.isinf(rs)] = 0.0
    left = sp.diags(rs)
    if mean_flag:
        return left * mat
    cs = np.asarray(mat.sum(0))
    cs = np.power(cs + 1e-8, -0.5).ravel()
    cs[np.isinf(cs)] = 0.0
    return left * mat * sp.diags(cs)


def to_torch_coo(mat: sp.spmatrix) -> torch.Tensor:
    """scipy -> torch sparse COO fp32 with int64 indices (main.py:105-112)."""
    coo = mat.tocoo()
    idx = torch.from_numpy(np.vstack((coo.row, coo.col)).astype(np.int64))
    val = torch.from_numpy(np.asarray(coo.data))
    return torch.sparse_coo_tensor(idx, val, torch.Size(coo.shape)).to(torch.float32)


def build_graphs(train_mat: sp.spmatrix) -> Tuple[torch.Tensor, torch.Tensor]:
    """ui_graph, iu_graph as Trainer.__init__ builds them (main.py:58,65-67)."""
    ui = to_torch_coo(csr_norm(train_mat, mean_flag=True))
    iu = to_torch_coo(csr_norm(train_mat.T, mean_flag=True))
    return ui, iu


# --------------------------------------------------------------------------------------
# parameters
# --------------------------------------------------------------------------------------
LIVE_PARAMS = ("image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias",
               "user_id_embedding.weight", "item_id_embedding.weight",
               "weight_dict.w_self_attention_cat", "weight_dict.w_q")


def xavier_uniform(shape: Sequence[int], gen: torch.Generator, dtype=torch.float32) -> torch.Tensor:
    fan_out, fan_in = shape[0], shape[1]
    bound = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(*shape, generator=gen, dtype=torch.float64) * 2 - 1).mul_(bound).to(dtype)


def init_params(n_users: int, n_items: int, dv: int, dt: int, cfg: HotPathConfig,
                seed: int = 2022, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Random parameters with the reference's init distributions (Models.py:28-31,41-45,58-66).
    (Values differ from ``torch.manual_seed``-driven init; parity tests load the same tensors on
    both sides instead of relying on RNG streams.)"""
    g = torch.Generator().manual_seed(seed)
    d = cfg.embed_size
    p = {
        "image_trans.weight": xavier_uniform((d, dv), g, dtype),
        "image_trans.bias": ((torch.rand(d, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(dv)).to(dtype),
        "text_trans.weight": xavier_uniform((d, dt), g, dtype),
        "text_trans.bias": ((torch.rand(d, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(dt)).to(dtype),
        "user_id_embedding.weight": xavier_uniform((n_users, d), g, dtype),
        "item_id_embedding.weight": xavier_uniform((n_items, d), g, dtype),
        "weight_dict.w_q": xavier_uniform((d, d), g, dtype),
        "weight_dict.w_k": xavier_uniform((d, d), g, dtype),
        "weight_dict.w_self_attention_cat": xavier_uniform((cfg.head_num * d, d), g, dtype),
    }
    return p


# --------------------------------------------------------------------------------------
# forward -- literal restatement  (Models.py:139-220)
# --------------------------------------------------------------------------------------
def _spmm(a: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    # Models.py:69-73 (args.sparse=1) and Models.py:203-208
    return torch.sparse.mm(a, x)


def _attention_literal(pair: Sequence[torch.Tensor], w_q: torch.Tensor, w_cat: torch.Tensor,
                       head_num: int, d: int) -> torch.Tensor:
    """Models.py:139-169.  `pair` = the two modality tensors [N,d] (dict order image, text).
    K is rebuilt from Q (:150) so w_k never participates; V is broadcast along the *query*
    modality axis (:154) so the softmax-weighted sum over keys returns V itself."""
    stacked = torch.stack(list(pair), dim=0)                       # :125-136  [2,N,d]
    n_mod, n_rows = stacked.shape[0], stacked.shape[1]
    dh = d / head_num                                              # :143 (a float)
    q = torch.matmul(stacked, w_q)                                 # :145
    q = q.reshape(n_mod, n_rows, head_num, int(dh)).permute(2, 0, 1, 3)   # :149
    k = q.reshape(n_mod, n_rows, head_num, int(dh)).permute(2, 0, 1, 3)   # :150 (from Q, post-permute)
    q = q.unsqueeze(2)                                             # :152
    k = k.unsqueeze(1)                                             # :153
    v = stacked.unsqueeze(1)                                       # :154
    att = torch.mul(q, k) / torch.sqrt(torch.tensor(dh))           # :156
    att = att.sum(dim=-1).unsqueeze(-1)                            # :157-158
    att = F.softmax(att, dim=2)                                    # :159
    z = torch.mul(att, v).sum(dim=2)                               # :161-162  [H,2,N,d]
    z = torch.cat([z[h] for h in range(z.shape[0])], dim=-1)       # :164-165  [2,N,H*d]
    return torch.matmul(z, w_cat)                                  # :166      [2,N,d]


def forward_literal(params: Dict[str, torch.Tensor], image_feats: torch.Tensor, text_feats: torch.Tensor,
                    graphs: Sequence[torch.Tensor], cfg: HotPathConfig,
                    dropout_masks: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                    training: bool = True):
    """Returns the reference's 12-tuple (Models.py:220).

    graphs = (ui, iu, image_ui, image_iu, text_ui, text_iu).
    dropout_masks: two [I,d] tensors holding 0 or 1/(1-p) (inverted-dropout scale); when None and
    training, torch's dropout op is used (consumes the global RNG like the reference)."""
    ui, iu, img_ui, img_iu, txt_ui, txt_iu = graphs
    d = cfg.embed_size

    def drop(x, which):
        if dropout_masks is not None:
            return x * dropout_masks[which]
        return F.dropout(x, p=cfg.drop_rate, training=training)

    xv = drop(F.linear(image_feats, params["image_trans.weight"], params["image_trans.bias"]), 0)  # :173
    xt = drop(F.linear(text_feats, params["text_trans.weight"], params["text_trans.bias"]), 1)     # :174
    e_u = params["user_id_embedding.weight"]
    e_i = params["item_id_embedding.weight"]

    for _ in range(cfg.feat_layers):                                # :176 (idempotent)
        u_v = _spmm(ui, xv)                                         # :177
        i_v = _spmm(iu, u_v)                                        # :178
        u_vid = _spmm(img_ui, e_i)                                  # :179
        i_vid = _spmm(img_iu, e_u)                                  # :180
        u_t = _spmm(ui, xt)                                         # :182
        i_t = _spmm(iu, u_t)                                        # :183
        u_tid = _spmm(txt_ui, e_i)                                  # :185
        i_tid = _spmm(txt_iu, e_u)                                  # :186

    w_q, w_cat = params["weight_dict.w_q"], params["weight_dict.w_self_attention_cat"]
    user_z = _attention_literal((u_vid, u_tid), w_q, w_cat, cfg.head_num, d)   # :192
    item_z = _attention_literal((i_vid, i_tid), w_q, w_cat, cfg.head_num, d)   # :193
    u = e_u + cfg.id_cat_rate * F.normalize(user_z.mean(0), p=2, dim=1)        # :194,196
    i = e_i + cfg.id_cat_rate * F.normalize(item_z.mean(0), p=2, dim=1)        # :195,197

    u_all, i_all = [u], [i]
    for layer in range(cfg.n_layers):                               # :201-211
        if layer == cfg.n_layers - 1:
            u = torch.softmax(torch.mm(ui, i), dim=-1)              # :203
            i = torch.softmax(torch.mm(iu, u), dim=-1)              # :204
        else:
            u = torch.mm(ui, i)                                     # :207
            i = torch.mm(iu, u)                                     # :208
        u_all.append(u)
        i_all.append(i)

    u_f = torch.stack(u_all).mean(dim=0)                            # :213
    i_f = torch.stack(i_all).mean(dim=0)                            # :214
    c = cfg.model_cat_rate
    u_f = u_f + c * F.normalize(u_v, p=2, dim=1) + c * F.normalize(u_t, p=2, dim=1)    # :217
    i_f = i_f + c * F.normalize(i_v, p=2, dim=1) + c * F.normalize(i_t, p=2, dim=1)    # :218
    return (u_f, i_f, i_v, i_t, u_v, u_t, u_f, i_f, u_vid, u_tid, i_vid, i_tid)        # :220


# --------------------------------------------------------------------------------------
# forward -- closed form (SURVEY.md appendix A); what the CUDA path computes
# --------------------------------------------------------------------------------------
def forward_closed(params, image_feats, text_feats, graphs, cfg: HotPathConfig,
                   dropout_masks=None, training: bool = True):
    ui, iu, img_ui, img_iu, txt_ui, txt_iu = graphs
    d, h = cfg.embed_size, cfg.head_num

    def drop(x, which):
        if dropout_masks is not None:
            return x * dropout_masks[which]
        return F.dropout(x, p=cfg.drop_rate, training=training)

    xv = drop(image_feats @ params["image_trans.weight"].t() + params["image_trans.bias"], 0)
    xt = drop(text_feats @ params["text_trans.weight"].t() + params["text_trans.bias"], 1)
    e_u, e_i = params["user_id_embedding.weight"], params["item_id_embedding.weight"]
    u_v = _spmm(ui, xv); i_v = _spmm(iu, u_v)
    u_t = _spmm(ui, xt); i_t = _spmm(iu, u_t)
    u_vid = _spmm(img_ui, e_i); i_vid = _spmm(img_iu, e_u)
    u_tid = _spmm(txt_ui, e_i); i_tid = _spmm(txt_iu, e_u)
    w_sum = params["weight_dict.w_self_attention_cat"].reshape(h, d, d).sum(0)
    u = e_u + cfg.id_cat_rate * F.normalize((0.5 * (u_vid + u_tid)) @ w_sum, dim=1)
    i = e_i + cfg.id_cat_rate * F.normalize((0.5 * (i_vid + i_tid)) @ w_sum, dim=1)
    s_u, s_i = u, i
    for layer in range(cfg.n_layers):
        u = _spmm(ui, i)
        if layer == cfg.n_layers - 1:
            u = torch.softmax(u, dim=-1)
        i = _spmm(iu, u)
        if layer == cfg.n_layers - 1:
            i = torch.softmax(i, dim=-1)
        s_u = s_u + u
        s_i = s_i + i
    c = cfg.model_cat_rate
    u_f = s_u / (cfg.n_layers + 1) + c * F.normalize(u_v, dim=1) + c * F.normalize(u_t, dim=1)
    i_f = s_i / (cfg.n_layers + 1) + c * F.normalize(i_v, dim=1) + c * F.normalize(i_t, dim=1)
    return (u_f, i_f, i_v, i_t, u_v, u_t, u_f, i_f, u_vid, u_tid, i_vid, i_tid)


# --------------------------------------------------------------------------------------
# losses
# --------------------------------------------------------------------------------------
def bpr_loss(u_b: torch.Tensor, p_b: torch.Tensor, n_b: torch.Tensor, cfg: HotPathConfig):
    """main.py:499-511.  Returns (mf_loss, emb_loss, reg_loss=0.0).  The regulariser divides by
    the *configured* batch size (main.py:504), not by len(u_b)."""
    pos = (u_b * p_b).sum(dim=1)
    neg = (u_b * n_b).sum(dim=1)
    reg = 0.5 * (u_b ** 2).sum() + 0.5 * (p_b ** 2).sum() + 0.5 * (n_b ** 2).sum()
    reg = reg / cfg.batch_size
    mf = -F.logsigmoid(pos - neg).mean()
    return mf, cfg.emb_decay * reg, 0.0


def infonce(z1: torch.Tensor, z2: torch.Tensor, cfg: HotPathConfig, block: int = 1024) -> torch.Tensor:
    """main.py:218-249 (sim at :211-216).  The j-loop concatenates over all column blocks, so the
    result is block-size independent; the 1e-8 is added to the *ratio*, inside the log (:244)."""
    n = z1.shape[0]
    n_blk = (n - 1) // block + 1
    a, b = F.normalize(z1), F.normalize(z2)
    out = []
    for bi in range(n_blk):
        rows = slice(bi * block, (bi + 1) * block)
        refl = torch.exp(a[rows] @ a.t() / cfg.tau)
        betw = torch.exp(a[rows] @ b.t() / cfg.tau)
        diag_b = betw[:, rows].diagonal()
        diag_r = refl[:, rows].diagonal()
        out.append(-torch.log(diag_b / (refl.sum(1) + betw.sum(1) - diag_r) + 1e-8))
    return torch.cat(out).mean()


def infonce_literal(z1, z2, cfg: HotPathConfig, block: int = 1024):
    """Same as ``infonce`` but with the reference's double loop and per-block re-normalisation
    (main.py:228-246) -- used by the CPU baseline so the op count matches."""
    n = z1.shape[0]
    n_blk = (n - 1) // block + 1
    idx = torch.arange(0, n)
    out = []
    for bi in range(n_blk):
        ri = idx[bi * block:(bi + 1) * block]
        refl_parts, betw_parts = [], []
        for bj in range(n_blk):
            rj = idx[bj * block:(bj + 1) * block]
            refl_parts.append(torch.exp(torch.mm(F.normalize(z1[ri]), F.normalize(z1[rj]).t()) / cfg.tau))
            betw_parts.append(torch.exp(torch.mm(F.normalize(z1[ri]), F.normalize(z2[rj]).t()) / cfg.tau))
        refl = torch.cat(refl_parts, dim=-1)
        betw = torch.cat(betw_parts, dim=-1)
        lo, hi = bi * block, (bi + 1) * block
        out.append(-torch.log(betw[:, lo:hi].diag() / (refl.sum(1) + betw.sum(1) - refl[:, lo:hi].diag()) + 1e-8))
    return torch.cat(out).mean()


def feat_reg(i_v, i_t, u_v, u_t, n_items: int, cfg: HotPathConfig) -> torch.Tensor:
    """main.py:252-257."""
    r = 0.5 * (i_v ** 2).sum() + 0.5 * (i_t ** 2).sum() + 0.5 * (u_v ** 2).sum() + 0.5 * (u_t ** 2).sum()
    return cfg.feat_reg_decay * (r / n_items)


def hot_loss(outs, users, pos, neg, n_items: int, cfg: HotPathConfig, literal: bool = False):
    """Hot-step loss: main.py:368-371, :408-414, :420 without the G_rate*G_lossf GAN term.
    Returns (total, dict of components)."""
    u_f, i_f, i_v, i_t, u_v, u_t, g_user, _, u_vid, u_tid, _, _ = outs
    users = torch.as_tensor(users, dtype=torch.long)
    pos = torch.as_tensor(pos, dtype=torch.long)
    neg = torch.as_tensor(neg, dtype=torch.long)
    mf, emb, reg = bpr_loss(u_f[users], i_f[pos], i_f[neg], cfg)
    fr = feat_reg(i_v, i_t, u_v, u_t, n_items, cfg)
    nce = infonce_literal if literal else infonce
    cl = nce(u_vid[users], g_user[users], cfg) + nce(u_tid[users], g_user[users], cfg)
    total = mf + emb + reg + fr + cfg.cl_rate * cl
    return total, {"mf": mf, "emb": emb, "feat_reg": fr, "cl": cl}


# --------------------------------------------------------------------------------------
# AdamW  (torch.optim.AdamW semantics, defaults betas=(0.9,0.999), eps=1e-8, wd=1e-2)
# --------------------------------------------------------------------------------------
def adamw_step(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int,
               lr: float, wd: float = 1e-2, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8):
    """One decoupled-weight-decay Adam update, in place; `step` is 1-based."""
    p.mul_(1.0 - lr * wd)
    m.mul_(b1).add_(g, alpha=1.0 - b1)
    v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
    bc1 = 1.0 - b1 ** step
    bc2 = 1.0 - b2 ** step
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-lr / bc1)


# --------------------------------------------------------------------------------------
# sampling  (utility/load_data.py:153-191) -- semantic restatement with a private RNG
# --------------------------------------------------------------------------------------
def sample_triples(train_csr: sp.csr_matrix, batch: int, rng: np.random.Generator):
    """B distinct users (when B <= #users with >=1 item), one uniform positive from the user's
    row, one uniform negative by rejection against the row (load_data.py:154-180)."""
    indptr, indices = train_csr.indptr, train_csr.indices
    deg = np.diff(indptr)
    exist = np.nonzero(deg > 0)[0]
    if batch <= train_csr.shape[0]:
        users = rng.choice(exist, size=batch, replace=False)
    else:
        users = rng.choice(exist, size=batch, replace=True)
    n_items = train_csr.shape[1]
    pos = np.empty(batch, np.int64)
    neg = np.empty(batch, np.int64)
    for k, u in enumerate(users):
        row = indices[indptr[u]:indptr[u + 1]]
        pos[k] = row[rng.integers(0, len(row))]
        while True:
            c = rng.integers(0, n_items)
            if c not in row:
                neg[k] = c
                break
    return users.astype(np.int64), pos, neg


# --------------------------------------------------------------------------------------
# one full hot step on CPU (the unit bench.py's cpu_baseline times)
# --------------------------------------------------------------------------------------
class CpuHotStep:
    """forward_literal + hot_loss + autograd backward + torch AdamW on the live parameters."""

    def __init__(self, params, image_feats, text_feats, graphs, n_items, cfg: HotPathConfig):
        self.cfg = cfg
        self.params = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        self.image_feats, self.text_feats = image_feats, text_feats
        self.graphs = graphs
        self.n_items = n_items
        self.opt = torch.optim.AdamW(list(self.params.values()), lr=cfg.lr)

    def step(self, users, pos, neg, dropout_masks=None) -> float:
        outs = forward_literal(self.params, self.image_feats, self.text_feats, self.graphs, self.cfg,
                               dropout_masks=dropout_masks, training=True)
        total, _ = hot_loss(outs, users, pos, neg, self.n_items, self.cfg, literal=True)
        self.opt.zero_grad()
        total.backward()
        self.opt.step()
        return float(total)
