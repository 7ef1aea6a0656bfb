"""CUDA backend of the GAN-side ops (csrc/gan.cu) -- the namespace ``mmssl_b200.gan`` is given as ``K`` in the product.
One function per op of tests/gan_ops_cpu.py (its specification), same names and argument meaning; outputs are allocated
here, every call goes through the C ABI and raises when the extension or a CUDA device is missing (no CPU fallback).
GEMMs: ``GEMM_IMPL = "tc"`` routes every product through the general-width wgmma kernel (csrc/gemm_wide.cu; operands
split into bf16 hi/lo pairs, K-major, by the same split kernels as the projection); ``"simt"`` is the fp32 CUDA-core GEMM.
"tc" is the default: gemm_wide.cu is parity-green on the H100 (tests/test_gpu_zzz_gemm_wide.py; its accumulation
passes are bounded) and the full iteration on it is about 3x faster than on the CUDA-core route at Baby (tools/fullstep_bench.py;
the H100 numbers are in DESIGN section 6); ``MMSSL_GAN_GEMM=simt`` or ``gan_ops.GEMM_IMPL`` switch.  ``"cublas"`` sends the same products to the vendor library through
``torch.mm`` / ``addmm`` (fp32, TF32 off): the library baseline the tensor-core kernel is measured against
(tools/fullstep_bench.py --gemm cublas), not the product path."""
from __future__ import annotations

import os
import weakref

import torch

GEMM_IMPL = os.environ.get("MMSSL_GAN_GEMM", "tc")

from . import _lib, ops
from ._lib import ptr, stream


def _L():
    return _lib.load(require_device=True)


def _c(t: torch.Tensor) -> torch.Tensor:
    assert t.is_cuda and t.dtype == torch.float32, "fp32 CUDA tensors only"
    return t if t.is_contiguous() else t.contiguous()


def _new(*shape, like):
    return torch.empty(*shape, dtype=torch.float32, device=like.device)


# ---- bf16 hi/lo operand splits of the Discriminator's weights are reused by every product of an iteration (W1 alone enters 6 of
# them, 100 MB of traffic per split at Baby); activations are split per call.  Only tensors registered as weights are cached;
# `adam` (the only writer of the weights on this path) drops the cache, `weights_changed()` does it for any other writer.
# The split of a registered weight always lands in the SAME pair of buffers (`_split_bufs`): inside a CUDA graph the iteration's
# first use of W1 reads what the previous replay's post-Adam split left there -- a Python-side cache that handed out fresh
# buffers per split made the captured graph read the warm-up iteration's buffers for ever (round 2, first hardware run of the
# captured full step on this route: gradient penalty 1.5e-3 off).
_weights = {}            # data_ptr -> weak reference to the registered tensor OBJECT (an address alone could be reused)
_split_cache = {}
_split_bufs = {}


def register_weights(tensors) -> None:
    for t in tensors:
        _weights[t.data_ptr()] = weakref.ref(t)


def weights_changed() -> None:
    _split_cache.clear()
    for k in [k for k, r in _weights.items() if r() is None]:
        del _weights[k]
        for b in [b for b in _split_bufs if b[0] == k]:
            del _split_bufs[b]


def refresh_weight_splits() -> None:
    """For writers of the registered weights other than `adam` (a checkpoint load, a test copying state in) when a captured
    graph is in use: recompute, IN PLACE, every split the graph reads (the graph itself only re-splits after its own Adam step)."""
    weights_changed()
    for (p_, shape, transposed) in list(_split_bufs):
        ref = _weights.get(p_)
        if ref is not None and ref() is not None:
            _split(ref(), transposed)


def _split(t, transposed: bool):
    ref = _weights.get(t.data_ptr())
    if ref is None or ref() is not t:
        return ops.split_bf16_t(t) if transposed else ops.split_bf16(t)
    key = (t.data_ptr(), tuple(t.shape), transposed, t._version)
    hit = _split_cache.get(key)
    if hit is None:
        bufs = _split_bufs.get(key[:3])
        hit = ops.split_bf16_t(t, out=bufs) if transposed else ops.split_bf16(t, out=bufs)
        _split_bufs[key[:3]] = hit
        _split_cache[key] = hit
    return hit


def mm(a, b, ta=False, tb=False, alpha=1.0):
    a, b = _c(a), _c(b)
    m = a.shape[1] if ta else a.shape[0]
    n = b.shape[0] if tb else b.shape[1]
    if GEMM_IMPL == "tc":
        k = a.shape[0] if ta else a.shape[1]
        a_hi, a_lo = _split(a, ta)                                             # [m][ceil8(k)], K-major
        b_hi, b_lo = _split(b, not tb)                                         # [n][ceil8(k)], K-major
        return ops.gemm_bf16x3_wide(a_hi, a_lo, b_hi, b_lo, m, n, k, _new(m, n, like=a), alpha=alpha)
    if GEMM_IMPL == "cublas":
        return torch.mm(a.t() if ta else a, b.t() if tb else b).mul_(alpha)
    if GEMM_IMPL != "simt":
        raise ValueError("gan_ops.GEMM_IMPL must be 'tc', 'simt' or 'cublas'")
    return ops.sgemm(a, b, _new(m, n, like=a), trans_a=ta, trans_b=tb, alpha=alpha)


def mm_acc(dst, a, b, ta=False, tb=False, alpha=1.0):
    """dst += alpha * op(a) @ op(b), accumulated in the GEMM epilogue (no temporary)."""
    a, b = _c(a), _c(b)
    assert dst.is_contiguous() and dst.dim() == 2
    m, n = dst.shape
    if GEMM_IMPL == "tc":
        k = a.shape[0] if ta else a.shape[1]
        a_hi, a_lo = _split(a, ta)
        b_hi, b_lo = _split(b, not tb)
        ops.gemm_bf16x3_wide(a_hi, a_lo, b_hi, b_lo, m, n, k, dst, alpha=alpha, accumulate=True)
    elif GEMM_IMPL == "cublas":
        dst.addmm_(a.t() if ta else a, b.t() if tb else b, alpha=alpha)
    else:
        ops.sgemm(a, b, dst, trans_a=ta, trans_b=tb, alpha=alpha, beta=1.0)


def gather_rows(table, users):
    table = _c(table)
    out = _new(users.numel(), table.shape[1], like=table)
    _lib.check(_L().mmssl_gan_gather_rows(ptr(table), table.stride(0), ptr(users), users.numel(), table.shape[1], ptr(out), stream()))
    return out


def scatter_add_rows(dst, users, src):
    assert dst.is_contiguous()
    src = _c(src)
    _lib.check(_L().mmssl_gan_scatter_add_rows(ptr(dst), dst.stride(0), ptr(users), users.numel(), dst.shape[1], ptr(src), stream()))


def colsum(x):
    x = _c(x)
    out = _new(x.shape[1], like=x)
    _lib.check(_L().mmssl_gan_colsum(ptr(x), x.shape[0], x.shape[1], ptr(out), stream()))
    return out


def add_scaled(acc, x, alpha):
    assert acc.is_contiguous() and acc.numel() == x.numel()
    x = _c(x)
    _lib.check(_L().mmssl_gan_add_scaled(ptr(acc), ptr(x), float(alpha), acc.numel(), stream()))


def bn_fwd(a, bias, gamma, beta, mask, running_mean, running_var):
    a, mask = _c(a), _c(mask)
    n, h = a.shape
    hout, ah, r = _new(n, h, like=a), _new(n, h, like=a), _new(h, like=a)
    _lib.check(_L().mmssl_gan_bn_fwd(ptr(a), ptr(bias), ptr(gamma), ptr(beta), ptr(mask), ptr(running_mean), ptr(running_var),
                                     n, h, ptr(hout), ptr(ah), ptr(r), stream()))
    return hout, ah, r


def bn_bwd(dh, mask, gamma, ah, r):
    dh = _c(dh)
    n, h = dh.shape
    da, dy, dg, db = _new(n, h, like=dh), _new(n, h, like=dh), _new(h, like=dh), _new(h, like=dh)
    _lib.check(_L().mmssl_gan_bn_bwd(ptr(dh), ptr(mask), ptr(gamma), ptr(ah), ptr(r), n, h, ptr(da), ptr(dy), ptr(dg), ptr(db), stream()))
    return da, dy, dg, db


def head_fwd(h2, w3, b3):
    h2 = _c(h2)
    n, h = h2.shape
    s, s_sum = _new(n, like=h2), _new(1, like=h2)
    _lib.check(_L().mmssl_gan_head_fwd(ptr(h2), ptr(w3), ptr(b3), n, h, ptr(s), ptr(s_sum), stream()))
    return s, s_sum


def head_bwd(s, coef, w3, h2):
    n, h = h2.shape
    dh2, dz, dw3, db3 = _new(n, h, like=h2), _new(n, like=h2), _new(h, like=h2), _new(1, like=h2)
    _lib.check(_L().mmssl_gan_head_bwd(ptr(s), float(coef), ptr(w3), ptr(h2), n, h, ptr(dh2), ptr(dz), ptr(dw3), ptr(db3), stream()))
    return dh2, dz, dw3, db3


def gp_rows(gx, lam):
    gx = _c(gx)
    n, w = gx.shape
    gbar, sq, gp = _new(n, w, like=gx), _new(n, like=gx), _new(1, like=gx)
    _lib.check(_L().mmssl_gan_gp_rows(ptr(gx), n, w, float(lam), ptr(gbar), ptr(sq), ptr(gp), stream()))
    return gp, gbar


def gp_rev_bn(q, dy, ah, r, gamma, mask):
    q = _c(q)
    n, h = q.shape
    dh_bar, ah_bar, r_bar, gg = _new(n, h, like=q), _new(n, h, like=q), _new(h, like=q), _new(h, like=q)
    _lib.check(_L().mmssl_gan_gp_rev_bn(ptr(q), ptr(dy), ptr(ah), ptr(r), ptr(gamma), ptr(mask), n, h, ptr(dh_bar), ptr(ah_bar),
                                        ptr(r_bar), ptr(gg), stream()))
    return dh_bar, ah_bar, r_bar, gg


def gp_head_rev(dh2_bar, dz, s, w3, h2):
    dh2_bar = _c(dh2_bar)
    n, h = dh2_bar.shape
    zb, h_bar, gw3, gb3 = _new(n, like=h2), _new(n, h, like=h2), _new(h, like=h2), _new(1, like=h2)
    _lib.check(_L().mmssl_gan_gp_head_rev(ptr(dh2_bar), ptr(dz), ptr(s), ptr(w3), ptr(h2), n, h, ptr(zb), ptr(h_bar), ptr(gw3),
                                          ptr(gb3), stream()))
    return h_bar, gw3, gb3


def bn_fwd_rev(h_bar, mask, gamma, ah, r, ah_bar, r_bar):
    h_bar = _c(h_bar)
    n, h = h_bar.shape
    a_bar, gg, gb = _new(n, h, like=h_bar), _new(h, like=h_bar), _new(h, like=h_bar)
    _lib.check(_L().mmssl_gan_bn_fwd_rev(ptr(h_bar), ptr(mask), ptr(gamma), ptr(ah), ptr(r), ptr(ah_bar), ptr(r_bar), n, h,
                                         ptr(a_bar), ptr(gg), ptr(gb), stream()))
    return a_bar, gg, gb


def usim_finish(scores, users, indptr, indices):
    scores = _c(scores)
    rows, w = scores.shape
    y, nrm = _new(rows, w, like=scores), _new(rows, like=scores)
    _lib.check(_L().mmssl_gan_usim_finish(ptr(scores), ptr(users), ptr(indptr), ptr(indices), rows, w, ptr(y), ptr(nrm), stream()))
    return y, nrm


def usim_bwd_pre(g, y, nrm, users, indptr, indices):
    g = _c(g)
    rows, w = g.shape
    out = _new(rows, w, like=g)
    _lib.check(_L().mmssl_gan_usim_bwd_pre(ptr(g), ptr(y), ptr(nrm), ptr(users), ptr(indptr), ptr(indices), rows, w, ptr(out), stream()))
    return out


def real_rows(users, indptr, indices, uniform, ui_sim, log_log_scale, tau, pre_scale):
    uniform, ui_sim = _c(uniform), _c(ui_sim)
    rows, w = uniform.shape
    out = _new(rows, w, like=uniform)
    _lib.check(_L().mmssl_gan_real_rows(ptr(users), ptr(indptr), ptr(indices), ptr(uniform), ptr(ui_sim), rows, w,
                                        float(log_log_scale), float(tau), float(pre_scale), ptr(out), stream()))
    return out


def interpolate(alpha, xr, xf):
    xr, xf = _c(xr), _c(xf)
    rows, w = xr.shape
    out = _new(rows, w, like=xr)
    _lib.check(_L().mmssl_gan_interpolate(ptr(_c(alpha)), ptr(xr), ptr(xf), rows, w, ptr(out), stream()))
    return out


def adam(params, grads, ms, vs, step, lr, b1, b2, eps=1e-8, step_dev=None):
    """torch.optim.Adam without weight decay == the library's AdamW kernel with weight_decay = 0.  ``step_dev`` (int32 device
    scalar holding step - 1) is advanced by a kernel, so the call is CUDA-graph capturable; without it the counter is uploaded
    from the host value (one small H2D copy per call)."""
    if step_dev is None:
        step_dev = torch.tensor([int(step)], dtype=torch.int32, device=params[0].device)
    else:
        ops.step_tick(step_dev)
    weights_changed()
    ops.adamw(list(params), [_c(g) for g in grads], list(ms), list(vs), step_dev, lr, b1, b2, eps, 0.0)
