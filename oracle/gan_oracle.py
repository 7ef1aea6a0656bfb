"""CPU oracle for the GAN side of the reference's training step (SURVEY.md section 8f row 2) and for the FULL step
(D step + G step) it is part of.  TEST INFRASTRUCTURE -- NOT PRODUCT CODE; only ``tests/`` may import it.

Restated on stock CPU torch, gradients by torch autograd -- the engine the reference itself uses (citations relative to
MMSSL/ of the reference repository):

  * u_sim_calculation            main.py:283-298   dense [B, I] scores, training items zeroed, rows L2-normalised
  * Discriminator                Models.py:224-245 Linear -> LeakyReLU(True) -> BatchNorm1d -> Dropout, twice, Linear -> Sigmoid, x100
  * weights_init                 main.py:135-138   (only documented: the tests start from recorded weights)
  * gradient_penalty             main.py:140-160   LAMBDA = 0.3, interpolation coefficient alpha ~ U(0,1) per row
  * D step                       main.py:339-361   fake = cat(image, text) similarity rows, real = Gumbel-perturbed interaction rows
  * G step                       main.py:363-429   hot-path loss + G_rate * (-mean D(cat(G_image_u_sim, G_text_u_sim)))
  * modality-graph bookkeeping   main.py:377-405   top-k ids collected at step 0, graphs rebuilt when idx % T == 0 and idx != 0
  * optimisers                   main.py:74 (Adam, lr D_lr, betas (0.5, 0.9)) and main.py:76-80 (AdamW defaults)

Quirks kept on purpose:
  * ``nn.LeakyReLU(True)`` passes True as *negative_slope* (= 1.0): the activation is the identity (Models.py:229,234);
  * BatchNorm1d runs in training mode in all four D calls of a step, also inside the gradient penalty (so the penalty's
    double backward goes through batch statistics) and in the G step (running stats move 4 times per step);
  * the (x, y) lists of the top-k graph update pair ``users`` TILED k times with the row-major flattened ids
    (main.py:398-399): entry j is (users[j % B], ids[j // k, j % k]) -- not (users[j // k], ...);
  * duplicates in those lists are summed by scipy, so rebuilt graphs hold values > 1 before normalisation; with the
    default m_topk_rate (1e-4) k = int(I * 1e-4) = 0 and the rebuilt graphs are empty.

PARITY PIN: ``tests/golden/gan_trace.npz`` -- a recorded trace of three steps of the unmodified ``Trainer.train()``
(``tests/golden/make_golden_gan.py``: D inputs/outputs, u_sim results, penalties, gradients, both optimisers' results,
rebuilt graphs, every random draw); ``tests/test_gan_oracle.py`` replays it through this file.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn.functional as F
from torch import autograd

from . import mmssl_oracle as O


@dataclass
class GanConfig:
    G_drop1: float = 0.31          # parser.py:84
    G_drop2: float = 0.5           # parser.py:85
    gp_rate: float = 1.0           # parser.py:86
    G_rate: float = 1e-4           # parser.py:83
    D_lr: float = 3e-4             # parser.py:56
    log_log_scale: float = 1e-5    # parser.py:99
    real_data_tau: float = 0.005   # parser.py:88
    ui_pre_scale: float = 100.0    # parser.py:89
    m_topk_rate: float = 1e-4      # parser.py:98
    T: int = 1                     # parser.py:93
    gp_lambda: float = 0.3         # main.py:142


# ------------------------------------------------------------------------------------------ u_sim
def u_sim(users: Sequence[int], user_final: torch.Tensor, item_final: torch.Tensor, train_csr: sp.csr_matrix,
          batch_size: int) -> torch.Tensor:
    """main.py:283-298 -- column blocks of `batch_size` items like the reference."""
    users = [int(u) for u in users]
    topk_u = user_final[users]
    u_ui = torch.from_numpy(np.asarray(train_csr[users].todense()))
    n_items = item_final.shape[0]
    parts = []
    for b in range((n_items - 1) // batch_size + 1):
        sl = slice(b * batch_size, (b + 1) * batch_size)
        sim = torch.mm(topk_u, item_final[sl].T)
        parts.append(sim * (1 - u_ui[:, sl]))
    return F.normalize(torch.cat(parts, dim=-1), p=2, dim=1)


# ------------------------------------------------------------------------------------------ Discriminator
D_PARAMS = ("net.0.weight", "net.0.bias", "net.2.weight", "net.2.bias", "net.4.weight", "net.4.bias", "net.6.weight",
            "net.6.bias", "net.8.weight", "net.8.bias")


def discriminator(x: torch.Tensor, S: Dict[str, torch.Tensor], mask1: Optional[torch.Tensor], mask2: Optional[torch.Tensor],
                  training: bool = True) -> torch.Tensor:
    """Models.py:224-245.  S = state dict (parameters + BatchNorm buffers; the buffers are updated in place in training
    mode exactly like nn.BatchNorm1d).  mask1/mask2: inverted-dropout masks (0 or 1/(1-p)); None in eval mode."""
    def bn(h, k):
        if training:
            S[f"net.{k}.num_batches_tracked"] += 1
        return F.batch_norm(h, S[f"net.{k}.running_mean"], S[f"net.{k}.running_var"], S[f"net.{k}.weight"], S[f"net.{k}.bias"],
                            training, 0.1, 1e-5)

    w1 = S["net.0.weight"]
    h = F.linear(x.float() if w1.dtype == torch.float32 else x.to(w1.dtype), w1, S["net.0.bias"])     # fp64 only in closed-form tests
    h = F.leaky_relu(h, negative_slope=1.0)               # nn.LeakyReLU(True): negative_slope = True
    h = bn(h, 2)
    h = h * mask1 if training else h
    h = F.linear(h, S["net.4.weight"], S["net.4.bias"])
    h = F.leaky_relu(h, negative_slope=1.0)
    h = bn(h, 6)
    h = h * mask2 if training else h
    h = torch.sigmoid(F.linear(h, S["net.8.weight"], S["net.8.bias"]))
    return (100 * h).view(-1)


def gradient_penalty(S, xr: torch.Tensor, xf: torch.Tensor, alpha: torch.Tensor, mask1, mask2, cfg: GanConfig) -> torch.Tensor:
    """main.py:140-160; alpha [2B, 1] is the recorded torch.rand draw."""
    xf, xr = xf.detach(), xr.detach()
    a = alpha.expand_as(xr)
    inter = (a * xr + (1 - a) * xf).requires_grad_()
    out = discriminator(inter, S, mask1, mask2)
    g = autograd.grad(outputs=out, inputs=inter, grad_outputs=torch.ones_like(out), create_graph=True, retain_graph=True,
                      only_inputs=True)[0]
    return ((g.norm(2, dim=1) - 1) ** 2).mean() * cfg.gp_lambda


def real_rows(users, train_csr: sp.csr_matrix, uniform: torch.Tensor, ui_sim: torch.Tensor, cfg: GanConfig) -> torch.Tensor:
    """main.py:348-351: Gumbel-perturbed softmax of the interaction rows + scaled similarity, row-normalised."""
    u_ui = torch.from_numpy(np.asarray(train_csr[[int(u) for u in users]].todense()))
    u_ui = F.softmax(u_ui - cfg.log_log_scale * torch.log(-torch.log(uniform + 1e-8) + 1e-8) / cfg.real_data_tau, dim=1)
    u_ui = u_ui + ui_sim * cfg.ui_pre_scale
    return F.normalize(u_ui, dim=1)


def d_step_grads(S, inputf: torch.Tensor, inputr: torch.Tensor, alpha: torch.Tensor, masks1, masks2, cfg: GanConfig):
    """loss_D of main.py:343-358 and its gradients by autograd, without the optimiser step, in the dtype of S's parameters.
    inputf / inputr: [2B, I] fake and real rows; alpha [2B] or [2B, 1]; masks1/masks2: the masks of the fake, real and
    penalty calls.  S is not modified.  Returns gp, the per-row outputs of the three calls, and a gradient per D parameter
    (zeros where autograd has none: net.8.bias does not reach the penalty)."""
    Sa = {k: (v.detach().clone().requires_grad_(True) if k in D_PARAMS else v.clone()) for k, v in S.items()}
    dt = Sa["net.0.weight"].dtype
    inputf, inputr, alpha = inputf.detach().to(dt), inputr.detach().to(dt), alpha.detach().to(dt).view(-1, 1)
    masks1, masks2 = [m.to(dt) for m in masks1], [m.to(dt) for m in masks2]
    outf = discriminator(inputf, Sa, masks1[0], masks2[0])
    outr = discriminator(inputr, Sa, masks1[1], masks2[1])
    a = alpha.expand_as(inputr)
    inter = (a * inputr + (1 - a) * inputf).requires_grad_()
    outi = discriminator(inter, Sa, masks1[2], masks2[2])
    gi = autograd.grad(outputs=outi, inputs=inter, grad_outputs=torch.ones_like(outi), create_graph=True, retain_graph=True,
                       only_inputs=True)[0]
    gp = ((gi.norm(2, dim=1) - 1) ** 2).mean() * cfg.gp_lambda
    loss = -outr.mean() + outf.mean() + cfg.gp_rate * gp
    grads = autograd.grad(loss, [Sa[k] for k in D_PARAMS], allow_unused=True)
    return dict(gp=gp.detach(), outs=(outf.detach(), outr.detach(), outi.detach()),
                grads={k: (g.detach() if g is not None else torch.zeros_like(Sa[k])) for k, g in zip(D_PARAMS, grads)})


def g_side_grads(S, x_image: torch.Tensor, x_text: torch.Tensor, mask1, mask2, cfg: GanConfig):
    """The G_rate * G_lossf term of main.py:414-420 on fixed rows: the D outputs and the gradients w.r.t. the image and the
    text rows, by autograd in the dtype of S's parameters.  S is not modified."""
    Sa = {k: v.detach().clone() for k, v in S.items()}
    dt = Sa["net.0.weight"].dtype
    B = x_image.shape[0]
    x = torch.cat((x_image.detach(), x_text.detach()), dim=0).to(dt).requires_grad_()
    out = discriminator(x, Sa, mask1.to(dt), mask2.to(dt))
    dx = autograd.grad(cfg.G_rate * -out.mean(), x)[0]
    return out.detach(), dx[:B], dx[B:]


def adam_step(p, g, m, v, step: int, lr: float, b1: float = 0.5, b2: float = 0.9, eps: float = 1e-8):
    """torch.optim.Adam (no weight decay), in place; main.py:74."""
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    denom = (v.sqrt() / math.sqrt(1 - b2 ** step)).add_(eps)
    p.addcdiv_(m, denom, value=-lr / (1 - b1 ** step))


# ------------------------------------------------------------------------------------------ graph bookkeeping
def topk_pairs(users, sim: torch.Tensor, n_items: int, cfg: GanConfig) -> Tuple[List[int], List[int]]:
    """main.py:397-399 (and :400-402): the x list tiles `users`, the y list is the row-major flattened top-k ids."""
    k = int(n_items * cfg.m_topk_rate)
    _, ids = torch.topk(sim.detach(), k, dim=-1)
    x = torch.tensor([int(u) for u in users]).repeat(1, k).view(-1).tolist()
    return x, ids.reshape(-1).tolist()


def rebuild_graphs(x: List[int], y: List[int], n_users: int, n_items: int,
                   dtype=torch.float32) -> Tuple[torch.Tensor, torch.Tensor]:
    """main.py:379-391 for one modality: (ui, iu) torch sparse graphs from the collected pairs (fp32 like the reference;
    float64 for a high-precision evaluation)."""
    vdt = np.float64 if dtype == torch.float64 else np.float32
    tmp = sp.csr_matrix((np.ones(len(x), vdt), (x, y)), shape=(n_users, n_items))
    return O.to_torch_coo(O.csr_norm(tmp, True), dtype), O.to_torch_coo(O.csr_norm(tmp.T, True), dtype)


# ------------------------------------------------------------------------------------------ the full step
class FullStep:
    """State + one `step()` = the body of the reference's batch loop (main.py:333-434) with every random draw injected."""

    def __init__(self, params: Dict[str, torch.Tensor], d_state: Dict[str, torch.Tensor], image_feats, text_feats,
                 train_csr: sp.csr_matrix, cfg: O.HotPathConfig, gcfg: GanConfig, dtype=torch.float32):
        """dtype: float32 (the reference's arithmetic) takes the inputs as given; float64 casts every floating-point input,
        state and graph, and is the yardstick the device's fp32 results are measured against.  The random draws passed to
        `step` are cast the same way."""
        wide = dtype != torch.float32
        cast = lambda v: v.to(dtype) if wide and v.is_floating_point() else v
        self.dtype = dtype
        self.P = {k: cast(v).clone() for k, v in params.items()}
        self.S = {k: cast(v).clone() for k, v in d_state.items()}
        self.feats = (cast(image_feats), cast(text_feats))
        self.R = train_csr.tocsr().astype(np.float64) if wide else train_csr.tocsr()
        self.U, self.I = self.R.shape
        self.cfg, self.g = cfg, gcfg
        ui, iu = O.build_graphs(self.R, dtype)
        self.graphs = [ui, iu, ui, iu, ui, iu]
        self.idx = 0
        self.index = {"image": ([], []), "text": ([], [])}
        self.live = [k for k in self.P if k not in ("weight_dict.w_q", "weight_dict.w_k")]
        self.mG = {k: torch.zeros_like(self.P[k]) for k in self.live}
        self.vG = {k: torch.zeros_like(self.P[k]) for k in self.live}
        self.mD = {k: torch.zeros_like(self.S[k]) for k in D_PARAMS}
        self.vD = {k: torch.zeros_like(self.S[k]) for k in D_PARAMS}

    def _forward(self, masks):
        return O.forward_literal(self.P, self.feats[0], self.feats[1], self.graphs, self.cfg, dropout_masks=masks, training=True)

    def step(self, users, pos, neg, model_masks, d_masks1, d_masks2, gumbel_u, alpha) -> Dict[str, object]:
        """model_masks: 4 [I,d] masks (2 per forward); d_masks1/2: 4 masks each (one per D call); returns a trace dict."""
        cfg, g, B = self.cfg, self.g, self.cfg.batch_size
        if self.dtype != torch.float32:
            c = lambda v: v.to(self.dtype)
            model_masks, d_masks1, d_masks2 = ([c(m) for m in ms] for ms in (model_masks, d_masks1, d_masks2))
            gumbel_u, alpha = c(gumbel_u), c(alpha)
        tr: Dict[str, object] = {"D_in": [], "D_out": [], "u_sim": []}
        users = [int(u) for u in users]

        def D(x, call):
            out = discriminator(x, self.S, d_masks1[call], d_masks2[call])
            tr["D_in"].append(x.detach().clone()); tr["D_out"].append(out.detach().clone())
            return out

        def usim(uf, itf):
            s = u_sim(users, uf, itf, self.R, B)
            tr["u_sim"].append(s.detach().clone())
            return s

        # ---------------- D step (main.py:339-361)
        with torch.no_grad():
            outs = self._forward((model_masks[0], model_masks[1]))
        ui_sim = usim(outs[0], outs[1]).detach()
        img_sim = usim(outs[4], outs[2]).detach()
        txt_sim = usim(outs[5], outs[3]).detach()
        for k in D_PARAMS:
            self.S[k].requires_grad_(True)
            self.S[k].grad = None
        inputf = torch.cat((img_sim, txt_sim), dim=0)
        lossf = D(inputf, 0).mean()
        rr = real_rows(users, self.R, gumbel_u, ui_sim, g)
        inputr = torch.cat((rr, rr), dim=0)
        lossr = -D(inputr, 1).mean()
        # the penalty's D call is the third of the step; record it through the same hook order as the reference
        a = alpha.expand_as(inputr)
        inter = (a * inputr.detach() + (1 - a) * inputf.detach()).requires_grad_()
        out_i = D(inter, 2)
        gi = autograd.grad(outputs=out_i, inputs=inter, grad_outputs=torch.ones_like(out_i), create_graph=True,
                           retain_graph=True, only_inputs=True)[0]
        gp = ((gi.norm(2, dim=1) - 1) ** 2).mean() * g.gp_lambda
        loss_D = lossr + lossf + g.gp_rate * gp
        grads = autograd.grad(loss_D, [self.S[k] for k in D_PARAMS], allow_unused=True)
        tr["gp"], tr["loss_D"] = gp.detach(), loss_D.detach()
        tr["Dgrad"] = {k: (gr.detach().clone() if gr is not None else None) for k, gr in zip(D_PARAMS, grads)}
        with torch.no_grad():
            for k, gr in zip(D_PARAMS, grads):
                self.S[k].requires_grad_(False)
                if gr is not None:
                    adam_step(self.S[k], gr, self.mD[k], self.vD[k], self.idx + 1, g.D_lr)
        tr["Dstate"] = {k: v.detach().clone() for k, v in self.S.items()}

        # ---------------- G step (main.py:363-429)
        for k in self.live:
            self.P[k].requires_grad_(True)
        outs = self._forward((model_masks[2], model_masks[3]))
        hot, parts = O.hot_loss(outs, users, pos, neg, self.I, cfg, literal=True)
        g_img = usim(outs[4], outs[2])
        g_txt = usim(outs[5], outs[3])
        if self.idx % g.T == 0 and self.idx != 0:          # main.py:378-394
            gi_ui, gi_iu = rebuild_graphs(*self.index["image"], self.U, self.I, self.dtype)
            gt_ui, gt_iu = rebuild_graphs(*self.index["text"], self.U, self.I, self.dtype)
            tr["graphs"] = [gi_ui, gt_ui, gi_iu, gt_iu]     # order of the reference's four conversions
            new_graphs = [self.graphs[0], self.graphs[1], gi_ui, gi_iu, gt_ui, gt_iu]
            self.index = {"image": ([], []), "text": ([], [])}
        else:                                               # main.py:396-402
            for key, s in (("image", g_img), ("text", g_txt)):
                x, y = topk_pairs(users, s, self.I, g)
                self.index[key][0].extend(x); self.index[key][1].extend(y)
            new_graphs = self.graphs
        G_lossf = -D(torch.cat((g_img, g_txt), dim=0), 3).mean()
        batch_loss = hot + g.G_rate * G_lossf
        grads = autograd.grad(batch_loss, [self.P[k] for k in self.live], allow_unused=True)
        tr["batch_loss"], tr["G_lossf"], tr["parts"] = batch_loss.detach(), G_lossf.detach(), {k: v.detach() for k, v in parts.items()}
        tr["Ggrad"] = {k: gr.detach().clone() for k, gr in zip(self.live, grads)}
        with torch.no_grad():
            for k, gr in zip(self.live, grads):
                self.P[k].requires_grad_(False)
                O.adamw_step(self.P[k], gr, self.mG[k], self.vG[k], self.idx + 1, cfg.lr, cfg.weight_decay)
        tr["Gparam"] = {k: self.P[k].detach().clone() for k in self.live}
        self.graphs = new_graphs
        self.idx += 1
        return tr


# ==========================================================================================
# Closed forms (no autograd) -- the arithmetic a CUDA implementation of the D step executes.
# Verified against the autograd versions above in tests/test_gan_oracle.py.
#
# One D call on n rows (training mode), h1 = I/4, h2 = I/8:
#   a1 = x W1^T + b1 ; BN: mu, r = (var_biased + eps)^-1/2, ah = (a - mu) r, y = gamma ah + beta ; h = y * M
#   a2 = h1 W2^T + b2 ; BN ; h2 ; z = h2 w3^T + b3 ; s = sigmoid(z) ; out = 100 s
# GEMM census per call (big = n x I x h1): forward 1 big; parameter gradients 1 big (dW1); input gradient 1 big (dx);
# gradient penalty = forward + input gradient + 3 big in the second-order sweep (gbar W1^T, da1^T gbar, abar1^T x).
# ==========================================================================================
_EPS = 1e-5


def d_forward_cache(x: torch.Tensor, S: Dict[str, torch.Tensor], m1: torch.Tensor, m2: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Forward of one training-mode D call keeping what the backward sweeps need (BatchNorm buffers are NOT touched)."""
    c: Dict[str, torch.Tensor] = {"x": x, "m1": m1, "m2": m2}
    h = x
    for li, (lin, bn, mask) in enumerate((("net.0", "net.2", m1), ("net.4", "net.6", m2)), start=1):
        a = h @ S[lin + ".weight"].T + S[lin + ".bias"]
        mu = a.mean(0)
        var = ((a - mu) ** 2).mean(0)
        r = (var + _EPS).rsqrt()
        ah = (a - mu) * r
        y = ah * S[bn + ".weight"] + S[bn + ".bias"]
        c[f"hin{li}"], c[f"r{li}"], c[f"ah{li}"] = h, r, ah
        h = y * mask
    c["h2"] = h
    z = h @ S["net.8.weight"].T + S["net.8.bias"]
    c["s"] = torch.sigmoid(z).view(-1)
    c["out"] = 100 * c["s"]
    return c


def _bn_bwd(dah: torch.Tensor, ah: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    return r * (dah - dah.mean(0) - ah * (dah * ah).mean(0))


def d_backward(c: Dict[str, torch.Tensor], S: Dict[str, torch.Tensor], dout: torch.Tensor, need_dx: bool = False):
    """First-order sweep: gradients of sum(dout * out) w.r.t. the D parameters (and x).  Also returns the per-layer
    pre-BatchNorm gradients the second-order sweep reuses."""
    g: Dict[str, torch.Tensor] = {}
    dz = (100 * c["s"] * (1 - c["s"]) * dout).unsqueeze(1)                       # [n, 1]
    g["net.8.weight"] = dz.T @ c["h2"]
    g["net.8.bias"] = dz.sum(0)
    dh = dz @ S["net.8.weight"]
    keep = {"dz": dz}
    for li, (lin, bn, mask) in ((2, ("net.4", "net.6", c["m2"])), (1, ("net.0", "net.2", c["m1"]))):
        dy = dh * mask
        g[bn + ".weight"] = (dy * c[f"ah{li}"]).sum(0)
        g[bn + ".bias"] = dy.sum(0)
        dah = dy * S[bn + ".weight"]
        da = _bn_bwd(dah, c[f"ah{li}"], c[f"r{li}"])
        g[lin + ".weight"] = da.T @ c[f"hin{li}"]
        g[lin + ".bias"] = da.sum(0)                                              # exactly 0 in exact arithmetic
        keep[f"dy{li}"], keep[f"dah{li}"], keep[f"da{li}"] = dy, dah, da
        if li == 2 or need_dx:
            dh = da @ S[lin + ".weight"]
    return g, (dh if need_dx else None), keep


def gradient_penalty_closed(x: torch.Tensor, S: Dict[str, torch.Tensor], m1, m2, lam: float = 0.3):
    """gp = lam * mean_i (||g_i|| - 1)^2 with g = d(sum out)/dx, and its gradient w.r.t. every D parameter,
    by an explicit reverse sweep over [forward ; first-order backward]."""
    n = x.shape[0]
    c = d_forward_cache(x, S, m1, m2)
    _, gx, k = d_backward(c, S, torch.ones(n), need_dx=True)
    norm = gx.norm(2, dim=1, keepdim=True)
    gp = lam * ((norm - 1) ** 2).mean()
    # d gp / d g  [n, I]; a zero row (saturated heads) gets torch's norm backward: 0, where the plain formula gives NaN
    gbar = torch.where(norm > 0, (2 * lam / n) * (norm - 1) / norm, torch.zeros_like(norm)) * gx
    G = {kk: torch.zeros_like(S[kk]) for kk in D_PARAMS}

    # ---- reverse of the first-order backward sweep (bottom-up: layer 1 first) ----
    def rev_bn_bwd(q, dah, ah, r):
        """da = r * u, u = dah - mean(dah) - ah * mean(dah * ah).  q = adjoint of da.
        Returns adjoints of (dah, ah, r)."""
        u = dah - dah.mean(0) - ah * (dah * ah).mean(0)
        r_bar = (q * u).sum(0)
        ub = q * r
        c_bar = -(ub * ah).sum(0) / n
        dah_bar = ub - ub.mean(0) + c_bar * ah
        ah_bar = c_bar * dah - ub * (dah * ah).mean(0)
        return dah_bar, ah_bar, r_bar

    q1 = gbar @ S["net.0.weight"].T                                              # adjoint of da1   (big GEMM)
    G["net.0.weight"] += k["da1"].T @ gbar                                       #                  (big GEMM)
    dah1_bar, ah1_bar, r1_bar = rev_bn_bwd(q1, k["dah1"], c["ah1"], c["r1"])
    G["net.2.weight"] += (dah1_bar * k["dy1"]).sum(0)
    dh1_bar = dah1_bar * S["net.2.weight"] * c["m1"]                             # adjoint of dh1 = da2 W2
    q2 = dh1_bar @ S["net.4.weight"].T
    G["net.4.weight"] += k["da2"].T @ dh1_bar
    dah2_bar, ah2_bar, r2_bar = rev_bn_bwd(q2, k["dah2"], c["ah2"], c["r2"])
    G["net.6.weight"] += (dah2_bar * k["dy2"]).sum(0)
    dh2_bar = dah2_bar * S["net.6.weight"] * c["m2"]                             # adjoint of dh2 = dz w3
    dz_bar = dh2_bar @ S["net.8.weight"].T                                       # [n, 1]
    G["net.8.weight"] += (k["dz"] * dh2_bar).sum(0, keepdim=True)
    s = c["s"].unsqueeze(1)
    s_bar = dz_bar * 100 * (1 - 2 * s)

    # ---- reverse of the forward sweep, seeded with the adjoints collected above ----
    z_bar = s_bar * s * (1 - s)
    G["net.8.weight"] += z_bar.T @ c["h2"]
    G["net.8.bias"] += z_bar.sum(0)
    h_bar = z_bar @ S["net.8.weight"]
    for li, (lin, bn, mask, ah_bar, r_bar) in ((2, ("net.4", "net.6", c["m2"], ah2_bar, r2_bar)),
                                               (1, ("net.0", "net.2", c["m1"], ah1_bar, r1_bar))):
        y_bar = h_bar * mask
        G[bn + ".weight"] += (y_bar * c[f"ah{li}"]).sum(0)
        G[bn + ".bias"] += y_bar.sum(0)
        ah_tot = ah_bar + y_bar * S[bn + ".weight"]
        a_bar = _bn_bwd(ah_tot, c[f"ah{li}"], c[f"r{li}"]) - (r_bar * c[f"r{li}"] ** 2) * c[f"ah{li}"] / n
        G[lin + ".weight"] += a_bar.T @ c[f"hin{li}"]                            # layer 1: big GEMM
        G[lin + ".bias"] += a_bar.sum(0)
        if li == 2:
            h_bar = a_bar @ S[lin + ".weight"]
    return gp, G


def u_sim_backward(users, user_final, item_final, train_csr: sp.csr_matrix, g_out: torch.Tensor):
    """Closed-form backward of u_sim: g_out [B, I] -> (rows of d user_final at `users` [B, d], d item_final [I, d])."""
    users = [int(u) for u in users]
    keep = 1 - torch.from_numpy(np.asarray(train_csr[users].todense()))
    ub = user_final[users]
    raw = (ub @ item_final.T) * keep
    nrm = raw.norm(2, dim=1, keepdim=True).clamp_min(1e-12)
    y = raw / nrm
    d_raw = (g_out - y * (g_out * y).sum(1, keepdim=True)) / nrm * keep
    return d_raw @ item_final, d_raw.T @ ub
