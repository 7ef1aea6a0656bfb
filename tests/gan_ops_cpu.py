"""Torch-CPU restatement of every device op `mmssl_b200/gan.py` sequences (one function per CUDA kernel of
`csrc/gan.cu`, same names, same argument meaning).  TEST INFRASTRUCTURE: it is the *specification* of those kernels --
the CPU suite injects it into the orchestration to check the sequencing against the reference trace, and the GPU suite
compares every CUDA op with the function of the same name here.  Not importable from the product."""
import torch

EPS = 1e-5
MOMENTUM = 0.1


def mm(a, b, ta=False, tb=False, alpha=1.0):
    return alpha * ((a.T if ta else a) @ (b.T if tb else b))


def mm_acc(dst, a, b, ta=False, tb=False, alpha=1.0):
    """dst += alpha * op(a) @ op(b)"""
    dst.add_(mm(a, b, ta, tb, alpha))


def gather_rows(table, users):
    return table[users]


def scatter_add_rows(dst, users, src):
    dst.index_add_(0, users, src)


def colsum(x):
    return x.sum(0)


def add_scaled(acc, x, alpha):
    acc.add_(x, alpha=alpha)


def bn_fwd(a, bias, gamma, beta, mask, running_mean, running_var):
    """Training-mode BatchNorm1d of (a + bias) followed by the dropout mask.  Returns h, ah (normalised), r (inverse std).
    Running statistics are updated in place (momentum 0.1, unbiased variance), like nn.BatchNorm1d."""
    n = a.shape[0]
    mu = a.mean(0)
    var = ((a - mu) ** 2).mean(0)
    r = (var + EPS).rsqrt()
    ah = (a - mu) * r
    running_mean.mul_(1 - MOMENTUM).add_(mu + bias, alpha=MOMENTUM)
    running_var.mul_(1 - MOMENTUM).add_(var * (n / (n - 1)), alpha=MOMENTUM)
    return (ah * gamma + beta) * mask, ah, r


def bn_bwd(dh, mask, gamma, ah, r):
    dy = dh * mask
    dah = dy * gamma
    da = r * (dah - dah.mean(0) - ah * (dah * ah).mean(0))
    return da, dy, (dy * ah).sum(0), dy.sum(0)


def head_fwd(h2, w3, b3):
    """s = sigmoid(h2 . w3 + b3); also sum(s) (the loss is +-100 * mean(s))."""
    s = torch.sigmoid(h2 @ w3.view(-1) + b3.view(()))
    return s, s.sum().view(1)


def head_bwd(s, coef, w3, h2):
    """Backward of sum(coef * 100 * s): dz, dh2 = dz (x) w3, dw3, db3."""
    dz = 100.0 * s * (1 - s) * coef
    return dz.unsqueeze(1) * w3.view(1, -1), dz, (dz.unsqueeze(1) * h2).sum(0), dz.sum().view(1)


def gp_rows(gx, lam):
    """A row with norm 0 gets a zero gradient, as torch's norm backward gives it (and still adds (0 - 1)^2 to gp)."""
    n = gx.shape[0]
    norm = gx.norm(2, dim=1, keepdim=True)
    gp = lam * ((norm - 1) ** 2).mean()
    f = torch.where(norm > 0, (2 * lam / n) * (norm - 1) / norm, torch.zeros_like(norm))
    return gp.view(1), f * gx


def gp_rev_bn(q, dy, ah, r, gamma, mask):
    """Adjoint of `da = bn_bwd(dh)` seeded with q = adjoint(da): returns adjoint(dh), adjoint(ah), adjoint(r) and the
    contribution to gamma's gradient."""
    n = q.shape[0]
    dah = dy * gamma
    cm = (dah * ah).mean(0)
    u = dah - dah.mean(0) - ah * cm
    r_bar = (q * u).sum(0)
    ub = q * r
    c_bar = -(ub * ah).sum(0) / n
    dah_bar = ub - ub.mean(0) + c_bar * ah
    ah_bar = c_bar * dah - ub * cm
    return dah_bar * gamma * mask, ah_bar, r_bar, (dah_bar * dy).sum(0)


def gp_head_rev(dh2_bar, dz, s, w3, h2):
    """Adjoint of the head's backward AND forward: returns adjoint(h2) from the forward, and the w3 / b3 gradients."""
    w = w3.view(-1)
    dz_bar = dh2_bar @ w
    s_bar = dz_bar * 100.0 * (1 - 2 * s)
    z_bar = s_bar * s * (1 - s)
    g_w3 = (dz.unsqueeze(1) * dh2_bar).sum(0) + (z_bar.unsqueeze(1) * h2).sum(0)
    return z_bar.unsqueeze(1) * w.view(1, -1), g_w3, z_bar.sum().view(1)


def bn_fwd_rev(h_bar, mask, gamma, ah, r, ah_bar, r_bar):
    """Adjoint of bn_fwd given adjoint(h) plus the extra adjoints of ah and r collected by gp_rev_bn."""
    n = h_bar.shape[0]
    y_bar = h_bar * mask
    tot = ah_bar + y_bar * gamma
    a_bar = r * (tot - tot.mean(0) - ah * (tot * ah).mean(0)) - (r_bar * r * r) * ah / n
    return a_bar, (y_bar * ah).sum(0), y_bar.sum(0)


def _keep(users, indptr, indices, n_items, dtype):
    keep = torch.ones(len(users), n_items, dtype=dtype)
    for k, u in enumerate(users.tolist()):
        keep[k, indices[indptr[u]:indptr[u + 1]]] = 0
    return keep


def usim_finish(scores, users, indptr, indices):
    raw = scores * _keep(users, indptr, indices, scores.shape[1], scores.dtype)
    nrm = raw.norm(2, dim=1).clamp_min(1e-12)
    return raw / nrm.unsqueeze(1), nrm


def usim_bwd_pre(g, y, nrm, users, indptr, indices):
    keep = _keep(users, indptr, indices, g.shape[1], g.dtype)
    return (g - y * (g * y).sum(1, keepdim=True)) / nrm.unsqueeze(1) * keep


def real_rows(users, indptr, indices, uniform, ui_sim, log_log_scale, tau, pre_scale):
    r = 1 - _keep(users, indptr, indices, uniform.shape[1], uniform.dtype)
    x = torch.softmax(r - log_log_scale * torch.log(-torch.log(uniform + 1e-8) + 1e-8) / tau, dim=1) + ui_sim * pre_scale
    return x / x.norm(2, dim=1, keepdim=True).clamp_min(1e-12)


def interpolate(alpha, xr, xf):
    a = alpha.view(-1, 1)
    return a * xr + (1 - a) * xf


def adam(params, grads, ms, vs, step, lr, b1, b2, eps=1e-8, step_dev=None):
    for p, g, m, v in zip(params, grads, ms, vs):
        m.mul_(b1).add_(g, alpha=1 - b1)
        v.mul_(b2).addcmul_(g, g, value=1 - b2)
        p.addcdiv_(m, (v.sqrt() / (1 - b2 ** step) ** 0.5).add_(eps), value=-lr / (1 - b1 ** step))
