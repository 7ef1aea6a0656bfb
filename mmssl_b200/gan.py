"""GAN side of the reference's training step (SURVEY 8f "next" #2): the Discriminator step and the generator-side
gradient, sequenced over device ops -- no autograd, no math in Python.

Reference: ``Discriminator`` (Models.py:224-245), ``u_sim_calculation`` (main.py:283-298), ``gradient_penalty``
(main.py:140-160), the D step (main.py:339-361) and the ``G_rate * G_lossf`` term of the G step (main.py:414-420).
The arithmetic is the closed form verified against autograd in ``oracle/gan_oracle.py`` (first-order sweep, the penalty's
second-order sweep through training-mode BatchNorm, u_sim backward).

Every function takes the op namespace ``K`` as first argument: ``mmssl_b200.gan_ops`` (CUDA kernels of csrc/gan.cu + the
library's GEMM; raises without the extension) in the product; the CPU suite injects a torch restatement of the same ops
(tests/gan_ops_cpu.py) to check the sequencing against the recorded reference trace.  One op == one kernel launch.

Reference quirks kept: ``nn.LeakyReLU(True)`` is the identity (negative_slope = True = 1.0) so it does not appear;
BatchNorm runs in training mode in all four D calls of a step; the biases in front of a BatchNorm get their (exactly zero,
numerically noisy) gradients like every other parameter because the reference's Adam updates them too.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import torch

PARAMS = ("net.0.weight", "net.0.bias", "net.2.weight", "net.2.bias", "net.4.weight", "net.4.bias", "net.6.weight",
          "net.6.bias", "net.8.weight", "net.8.bias")
BUFFERS = ("net.2.running_mean", "net.2.running_var", "net.2.num_batches_tracked", "net.6.running_mean", "net.6.running_var",
           "net.6.num_batches_tracked")


@dataclass
class GanHyper:
    gp_rate: float = 1.0           # parser.py:86
    gp_lambda: float = 0.3         # main.py:142
    G_rate: float = 1e-4           # parser.py:83
    D_lr: float = 3e-4             # parser.py:56
    beta1: float = 0.5             # main.py:74
    beta2: float = 0.9
    log_log_scale: float = 1e-5    # parser.py:99
    real_data_tau: float = 0.005   # parser.py:88
    ui_pre_scale: float = 100.0    # parser.py:89


class DiscriminatorState:
    """Parameters + BatchNorm buffers of the reference's ``Discriminator(n_items)`` under their state_dict names, plus the
    Adam moments of ``optim_D``."""

    def __init__(self, state: Dict[str, torch.Tensor]):
        self.t = {k: state[k] for k in PARAMS + BUFFERS}
        self.m = {k: torch.zeros_like(self.t[k]) for k in PARAMS}
        self.v = {k: torch.zeros_like(self.t[k]) for k in PARAMS}
        self.step = 0
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=self.t[PARAMS[0]].device)     # the same count, on the device

    def state_dict(self) -> Dict[str, torch.Tensor]:
        return dict(self.t)

    def optim_state_dict(self) -> Dict[str, object]:
        """Adam state of ``optim_D``: moments and the step count (host and device copies are the same number)."""
        return dict(m=dict(self.m), v=dict(self.v), step=int(self.step), step_dev=int(self.step_dev.cpu()[0]))

    def load_state_dict(self, state: Dict[str, torch.Tensor], optim: Optional[Dict[str, object]] = None) -> None:
        """Copies a ``Discriminator`` state_dict (and, when given, ``optim_state_dict()``) into the live tensors in place.
        Callers that use the tensor-core GEMM route refresh the cached weight splits afterwards (gan_ops.refresh_weight_splits)."""
        from .checkpoint import copy_into
        if optim is not None and int(optim["step"]) != int(optim["step_dev"]):
            raise ValueError(f"checkpoint mismatch in D step: host {optim['step']}, device {optim['step_dev']}")
        copy_into(self.t, state, "D")
        if optim is not None:
            copy_into(self.m, optim["m"], "D_optim.m")
            copy_into(self.v, optim["v"], "D_optim.v")
            self.step = int(optim["step"])
            self.step_dev.fill_(self.step)

    def zeros_like_params(self) -> Dict[str, torch.Tensor]:
        return {k: torch.zeros_like(self.t[k]) for k in PARAMS}


# ------------------------------------------------------------------------------------------ one D call
def d_forward(K, D: DiscriminatorState, x: torch.Tensor, m1: torch.Tensor, m2: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Training-mode forward on n rows; keeps what the backward sweeps need.  c['s_sum'] = sum(sigmoid) (out = 100 s)."""
    t = D.t
    a1 = K.mm(x, t["net.0.weight"], tb=True)
    h1, ah1, r1 = K.bn_fwd(a1, t["net.0.bias"], t["net.2.weight"], t["net.2.bias"], m1, t["net.2.running_mean"], t["net.2.running_var"])
    a2 = K.mm(h1, t["net.4.weight"], tb=True)
    h2, ah2, r2 = K.bn_fwd(a2, t["net.4.bias"], t["net.6.weight"], t["net.6.bias"], m2, t["net.6.running_mean"], t["net.6.running_var"])
    t["net.2.num_batches_tracked"] += 1
    t["net.6.num_batches_tracked"] += 1
    s, s_sum = K.head_fwd(h2, t["net.8.weight"], t["net.8.bias"])
    return dict(x=x, m1=m1, m2=m2, h1=h1, ah1=ah1, r1=r1, h2=h2, ah2=ah2, r2=r2, s=s, s_sum=s_sum)


def d_backward(K, D: DiscriminatorState, c: Dict[str, torch.Tensor], coef: float, grads: Optional[Dict[str, torch.Tensor]],
               scale: float = 1.0, need_dx: bool = False, keep: Optional[dict] = None) -> Optional[torch.Tensor]:
    """Backward of ``sum(coef * out)``.  Parameter gradients are added into ``grads`` (times ``scale``) unless it is None;
    returns d/dx when asked.  ``keep`` (a dict) receives dz, dy*, da* for the second-order sweep."""
    t = D.t
    dh2, dz, dw3, db3 = K.head_bwd(c["s"], coef, t["net.8.weight"], c["h2"])
    da2, dy2, dg2, dbe2 = K.bn_bwd(dh2, c["m2"], t["net.6.weight"], c["ah2"], c["r2"])
    dh1 = K.mm(da2, t["net.4.weight"])
    da1, dy1, dg1, dbe1 = K.bn_bwd(dh1, c["m1"], t["net.2.weight"], c["ah1"], c["r1"])
    if grads is not None:
        for k, g in (("net.8.weight", dw3.view_as(t["net.8.weight"])), ("net.8.bias", db3), ("net.6.weight", dg2), ("net.6.bias", dbe2),
                     ("net.4.bias", K.colsum(da2)), ("net.2.weight", dg1), ("net.2.bias", dbe1), ("net.0.bias", K.colsum(da1))):
            K.add_scaled(grads[k], g, scale)
        # the two weight gradients accumulate in the GEMM epilogue: no [I/4, I] temporary, no extra pass over it
        K.mm_acc(grads["net.4.weight"], da2, c["h1"], ta=True, alpha=scale)
        K.mm_acc(grads["net.0.weight"], da1, c["x"], ta=True, alpha=scale)
    if keep is not None:
        keep.update(dz=dz, dy2=dy2, da2=da2, dy1=dy1, da1=da1)
    return K.mm(da1, t["net.0.weight"]) if need_dx else None


def gradient_penalty(K, D: DiscriminatorState, inter: torch.Tensor, m1, m2, lam: float, grads: Dict[str, torch.Tensor],
                     scale: float) -> torch.Tensor:
    """gp = lam * mean_i (||d sum(out) / d x_i|| - 1)^2 on the interpolates; adds scale * d gp / d theta into ``grads``.
    Sequence = oracle/gan_oracle.py:gradient_penalty_closed (5 GEMMs of the n x I x I/4 size)."""
    t = D.t
    c = d_forward(K, D, inter, m1, m2)
    k: dict = {}
    gx = d_backward(K, D, c, 1.0, None, need_dx=True, keep=k)
    gp, gbar = K.gp_rows(gx, lam)
    # reverse of the first-order backward sweep
    q1 = K.mm(gbar, t["net.0.weight"], tb=True)
    K.mm_acc(grads["net.0.weight"], k["da1"], gbar, ta=True, alpha=scale)
    dh1_bar, ah1_bar, r1_bar, gg1 = K.gp_rev_bn(q1, k["dy1"], c["ah1"], c["r1"], t["net.2.weight"], c["m1"])
    K.add_scaled(grads["net.2.weight"], gg1, scale)
    q2 = K.mm(dh1_bar, t["net.4.weight"], tb=True)
    K.mm_acc(grads["net.4.weight"], k["da2"], dh1_bar, ta=True, alpha=scale)
    dh2_bar, ah2_bar, r2_bar, gg2 = K.gp_rev_bn(q2, k["dy2"], c["ah2"], c["r2"], t["net.6.weight"], c["m2"])
    K.add_scaled(grads["net.6.weight"], gg2, scale)
    # reverse of the forward sweep, seeded with the adjoints collected above
    h_bar, gw3, gb3 = K.gp_head_rev(dh2_bar, k["dz"], c["s"], t["net.8.weight"], c["h2"])
    K.add_scaled(grads["net.8.weight"], gw3.view_as(t["net.8.weight"]), scale)
    K.add_scaled(grads["net.8.bias"], gb3, scale)
    a2_bar, gg2b, gbe2 = K.bn_fwd_rev(h_bar, c["m2"], t["net.6.weight"], c["ah2"], c["r2"], ah2_bar, r2_bar)
    K.add_scaled(grads["net.6.weight"], gg2b, scale)
    K.add_scaled(grads["net.6.bias"], gbe2, scale)
    K.mm_acc(grads["net.4.weight"], a2_bar, c["h1"], ta=True, alpha=scale)
    K.add_scaled(grads["net.4.bias"], K.colsum(a2_bar), scale)
    h1_bar = K.mm(a2_bar, t["net.4.weight"])
    a1_bar, gg1b, gbe1 = K.bn_fwd_rev(h1_bar, c["m1"], t["net.2.weight"], c["ah1"], c["r1"], ah1_bar, r1_bar)
    K.add_scaled(grads["net.2.weight"], gg1b, scale)
    K.add_scaled(grads["net.2.bias"], gbe1, scale)
    K.mm_acc(grads["net.0.weight"], a1_bar, c["x"], ta=True, alpha=scale)
    K.add_scaled(grads["net.0.bias"], K.colsum(a1_bar), scale)
    return gp


# ------------------------------------------------------------------------------------------ u_sim
def u_sim_forward(K, user_final, item_final, users, indptr, indices) -> Dict[str, torch.Tensor]:
    """main.py:283-298: scores of the batch users against all items, training items zeroed, rows L2-normalised."""
    ub = K.gather_rows(user_final, users)
    y, nrm = K.usim_finish(K.mm(ub, item_final, tb=True), users, indptr, indices)
    return dict(y=y, nrm=nrm, ub=ub, users=users)


def u_sim_backward(K, c: Dict[str, torch.Tensor], g: torch.Tensor, item_final, indptr, indices, g_user_final, g_item_final) -> None:
    """Adds the gradients of ``sum(g * u_sim)`` into the full [U, d] / [I, d] gradient tables."""
    d_raw = K.usim_bwd_pre(g, c["y"], c["nrm"], c["users"], indptr, indices)
    K.scatter_add_rows(g_user_final, c["users"], K.mm(d_raw, item_final))
    K.mm_acc(g_item_final, d_raw, c["ub"], ta=True, alpha=1.0)


# ------------------------------------------------------------------------------------------ the two entry points
def d_step(K, D: DiscriminatorState, hp: GanHyper, image_sim, text_sim, ui_sim, users, indptr, indices, gumbel_u, alpha,
           masks1: Sequence[torch.Tensor], masks2: Sequence[torch.Tensor]) -> Dict[str, torch.Tensor]:
    """main.py:343-361.  *_sim: detached [B, I] u_sim rows; gumbel_u [B, I] ~ U(0,1); alpha [2B] ~ U(0,1);
    masks1/masks2: three inverted-dropout masks each ([2B, I/4], [2B, I/8]) for the fake, real and penalty calls."""
    n = 2 * image_sim.shape[0]
    grads = D.zeros_like_params()
    inputf = torch.cat((image_sim, text_sim), dim=0)
    cf = d_forward(K, D, inputf, masks1[0], masks2[0])                       # lossf = mean(out)
    d_backward(K, D, cf, 1.0 / n, grads)
    rr = K.real_rows(users, indptr, indices, gumbel_u, ui_sim, hp.log_log_scale, hp.real_data_tau, hp.ui_pre_scale)
    inputr = torch.cat((rr, rr), dim=0)
    cr = d_forward(K, D, inputr, masks1[1], masks2[1])                       # lossr = -mean(out)
    d_backward(K, D, cr, -1.0 / n, grads)
    inter = K.interpolate(alpha, inputr, inputf)
    gp = gradient_penalty(K, D, inter, masks1[2], masks2[2], hp.gp_lambda, grads, hp.gp_rate)
    D.step += 1
    K.adam([D.t[k] for k in PARAMS], [grads[k] for k in PARAMS], [D.m[k] for k in PARAMS], [D.v[k] for k in PARAMS], D.step,
           hp.D_lr, hp.beta1, hp.beta2, step_dev=D.step_dev)
    return dict(gp=gp, lossf_sum=cf["s_sum"], lossr_sum=cr["s_sum"], grads=grads, n=n)


def g_side(K, D: DiscriminatorState, hp: GanHyper, image_c: Dict[str, torch.Tensor], text_c: Dict[str, torch.Tensor], m1, m2):
    """The ``G_rate * G_lossf`` term (main.py:414-420): G_lossf = -mean(D(cat(G_image_u_sim, G_text_u_sim))).
    Returns (sum of sigmoid outputs, gradient w.r.t. the image rows, w.r.t. the text rows), the gradients already scaled by
    G_rate.  D's own gradients of this call are never used by the reference (zeroed before the next D backward)."""
    x = torch.cat((image_c["y"], text_c["y"]), dim=0)
    n, B = x.shape[0], image_c["y"].shape[0]
    c = d_forward(K, D, x, m1, m2)
    dx = d_backward(K, D, c, -hp.G_rate / n, None, need_dx=True)
    return c["s_sum"], dx[:B], dx[B:]
