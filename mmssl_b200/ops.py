"""Thin tensor-level wrappers over the C ABI (include/mmssl_b200.h).  No arithmetic happens here:
every function validates, allocates outputs with torch (device memory plumbing) and launches the
library kernels on torch's current CUDA stream."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import torch

from . import _lib
from ._lib import SpmmRhs, ptr, stream
from .graph import SparseOperand

EPI_NONE, EPI_SOFTMAX, EPI_SOFTMAX_BWD = 0, 1, 2
SPMM_IMPL_LDG, SPMM_IMPL_TMA = 0, 1     # TMA = shared-memory hot rows staged by cp.async.bulk (large graphs)
SPMM_IMPL_PIPE = 512          # software-pipelined walk of the plan by one resident wave (small graphs; | 64: early operand prefetch)
SPMM_IMPL_BULK = 0x100000               # staged gather pipeline (csrc/spmm_bulk.cu); low 20 bits = its variant word
SPMM_BULK_TMA = 0x10000                 # ... with one TMA bulk copy per neighbour row instead of warp-wide 16-byte cp.async
_default_spmm_impl = SPMM_IMPL_LDG
_small_spmm_impl = int(os.environ.get("MMSSL_SPMM_SMALL_IMPL", "0"), 0)     # experiment knob: impl for graphs under 2^21 non-zeros


def set_default_spmm_impl(impl: int) -> None:
    global _default_spmm_impl
    _default_spmm_impl = int(impl)


def _lib_() -> C.CDLL:
    return _lib.load(require_device=True)


def _row_ok(t: torch.Tensor) -> None:
    if t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1 or t.stride(0) % 4 != 0 or t.data_ptr() % 16 != 0:
        raise ValueError("expected a 2-D fp32 CUDA tensor with unit column stride, row stride % 4 == 0 and 16-byte alignment")
    if not t.is_cuda:
        raise _lib.MmsslLibraryError("mmssl_b200 operators only run on CUDA tensors (no CPU fallback)")


def _ld(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else int(t.stride(0))


def spmm(a: SparseOperand, xs: Sequence[torch.Tensor], ys: Optional[Sequence[torch.Tensor]] = None, *,
         epilogue: int = EPI_NONE, alpha: float = 1.0, cs: Optional[Sequence[Optional[torch.Tensor]]] = None,
         ysaved: Optional[Sequence[torch.Tensor]] = None, ss: Optional[Sequence[Optional[torch.Tensor]]] = None,
         s_mode: int = 0, sbases: Optional[Sequence[Optional[torch.Tensor]]] = None,
         impl: Optional[int] = None, y_mode: int = 0, y_raw: Optional[Sequence[int]] = None,
         y_peers: Optional[Sequence[Sequence[int]]] = None) -> List[torch.Tensor]:
    """Y_r = epi(A @ X_r + alpha * C_r), optional running sums; see mmssl_spmm_csr_f32.
    Fused all-gather (row-sharded tables): y_mode=1 with y_raw[r] = multicast address of the rank's row block
    (ys[r] = the local view of the same rows, used for shape/stride only), or y_mode=2 with y_peers[r] = the
    peer-mapped addresses of that row block on the other ranks."""
    lib = _lib_()
    nrhs = len(xs)
    d = xs[0].shape[1]
    if ys is None:
        ys = [torch.empty(a.n_rows, d, dtype=torch.float32, device=xs[0].device) for _ in range(nrhs)]
    rhs = (SpmmRhs * nrhs)()
    for r in range(nrhs):
        x, y = xs[r], ys[r]
        _row_ok(x); _row_ok(y)
        if x.shape != (a.n_cols, d) or y.shape != (a.n_rows, d):
            raise ValueError(f"spmm shape mismatch: A {a.n_rows}x{a.n_cols}, X {tuple(x.shape)}, Y {tuple(y.shape)}")
        c = cs[r] if cs is not None else None
        yv = ysaved[r] if ysaved is not None else None
        s = ss[r] if ss is not None else None
        sb = sbases[r] if sbases is not None else None
        for t in (c, yv, s, sb):
            if t is not None:
                _row_ok(t)
        rhs[r] = SpmmRhs(ptr(x), _ld(x), ptr(y), _ld(y), ptr(c), _ld(c), ptr(yv), _ld(yv), ptr(s), _ld(s), ptr(sb), _ld(sb))
        if y_mode == 1:
            rhs[r].y = int(y_raw[r])
            rhs[r].y_mode = 1
        elif y_mode == 2:
            rhs[r].y_mode = 2
            rhs[r].n_peers = len(y_peers[r])
            for k, pp in enumerate(y_peers[r]):
                rhs[r].y_peers[k] = int(pp)
    # split-row work area (partial sums + arrival counters), private to (operand, total width): launches
    # of different widths may run concurrently on two streams, and heavy rows need zeroed slots
    if impl is None:
        impl = _small_spmm_impl if (_small_spmm_impl and a.nnz < (1 << 21)) else _default_spmm_impl
    if impl & SPMM_IMPL_BULK and nrhs <= 2 and not (epilogue == EPI_SOFTMAX_BWD and s_mode != 0):
        b = a.bulk_plan()
        part, counters = a.bulk_work_area(nrhs * d)
        desc = type(b["desc"]).from_buffer_copy(b["desc"])
        desc.counters = counters.data_ptr()
        _lib.check(lib.mmssl_spmm_bulk_f32(C.byref(desc), ptr(b["buckets"]), b["n_buckets"], d, nrhs, rhs, epilogue, float(alpha),
                                           s_mode, ptr(part), part.numel(), impl & 0xfffff, stream()))
        return list(ys)
    if impl & SPMM_IMPL_BULK:
        impl = 0
    part, counters = a.work_area(nrhs * d)
    desc = type(a.desc).from_buffer_copy(a.desc)
    desc.counters = counters.data_ptr()
    if impl & 256:       # L1 hot / cold rows: the column indices carry the hot flag (about 192 KB of rows per SM)
        desc.colidx = a.hot_flag_colidx(max(1, (192 * 1024) // (nrhs * d * 4))).data_ptr()
    if impl == SPMM_IMPL_TMA:
        colidx_hot, hot_ids, n_hot = a.hot_plan()
        _lib.check(lib.mmssl_spmm_hot_f32(C.byref(desc), ptr(colidx_hot), ptr(hot_ids), n_hot, d, nrhs, rhs, epilogue,
                                          float(alpha), s_mode, ptr(part), part.numel(), stream()))
    else:
        _lib.check(lib.mmssl_spmm_csr_f32(C.byref(desc), d, nrhs, rhs, epilogue, float(alpha), s_mode, ptr(part),
                                          part.numel(), impl, stream()))
    return list(ys)


def sgemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, trans_a=False, trans_b=False, alpha=1.0, beta=0.0,
          split_k: int = 1) -> torch.Tensor:
    lib = _lib_()
    m = a.shape[1] if trans_a else a.shape[0]
    k = a.shape[0] if trans_a else a.shape[1]
    n = b.shape[0] if trans_b else b.shape[1]
    kb = b.shape[1] if trans_b else b.shape[0]
    assert k == kb and out.shape == (m, n), (a.shape, b.shape, out.shape, trans_a, trans_b)
    for t in (a, b, out):
        assert t.dtype == torch.float32 and t.stride(1) == 1 and t.is_cuda
    _lib.check(lib.mmssl_sgemm(int(trans_a), int(trans_b), m, n, k, float(alpha), ptr(a), a.stride(0), ptr(b), b.stride(0),
                               float(beta), ptr(out), out.stride(0), split_k, stream()))
    return out


def id_fuse_fwd(z, e, rate: float, out):
    lib = _lib_()
    n, d = z.shape
    zn = torch.empty(n, d, dtype=torch.float32, device=z.device)
    nrm = torch.empty(n, dtype=torch.float32, device=z.device)
    _lib.check(lib.mmssl_id_fuse_fwd(ptr(z), _ld(z), ptr(e), _ld(e), n, d, float(rate), ptr(out), _ld(out), ptr(zn), ptr(nrm), stream()))
    return out, zn, nrm


def id_fuse_bwd(g, zn, nrm, rate: float, dz):
    lib = _lib_()
    n, d = g.shape
    _lib.check(lib.mmssl_id_fuse_bwd(ptr(g), _ld(g), ptr(zn), ptr(nrm), n, d, float(rate), ptr(dz), _ld(dz), stream()))
    return dz


def wsum(wcat, d: int, heads: int):
    out = torch.empty(2, d, d, dtype=torch.float32, device=wcat.device)
    _lib.check(_lib_().mmssl_wsum(ptr(wcat), d, heads, ptr(out[0]), ptr(out[1]), stream()))
    return out[0], out[1]          # Wsum, Wsum^T


def id_fuse2_fwd(ya, yb, coef: float, w, e, rate: float):
    """out = e + rate * normalize(coef*(ya [+ yb]) @ w); returns (out, zn, nrm)."""
    lib = _lib_()
    n, d = ya.shape
    f = dict(dtype=torch.float32, device=ya.device)
    out, zn, nrm = torch.empty(n, d, **f), torch.empty(n, d, **f), torch.empty(n, **f)
    _lib.check(lib.mmssl_id_fuse2_fwd(ptr(ya), _ld(ya), ptr(yb), _ld(yb), float(coef), ptr(w), ptr(e), _ld(e), n, d, float(rate),
                                      ptr(out), _ld(out), ptr(zn), ptr(nrm), stream()))
    return out, zn, nrm


def id_fuse2_bwd(g, zn, nrm, ya, yb, coef: float, w_t, rate: float, ext_a, ext_b, two_outputs: bool):
    """Returns (out_a, out_b or None, dw_partials[blocks, d*d])."""
    lib = _lib_()
    n, d = g.shape
    f = dict(dtype=torch.float32, device=g.device)
    nb = lib.mmssl_id_fuse2_blocks(n)
    part = torch.empty(nb, d * d, **f)
    out_a = torch.empty(n, d, **f)
    out_b = torch.empty(n, d, **f) if two_outputs else None
    _lib.check(lib.mmssl_id_fuse2_bwd(ptr(g), _ld(g), ptr(zn), ptr(nrm), ptr(ya), _ld(ya), ptr(yb), _ld(yb), float(coef), ptr(w_t), n, d,
                                      float(rate), ptr(ext_a), _ld(ext_a), ptr(ext_b), _ld(ext_b), ptr(out_a), _ld(out_a),
                                      ptr(out_b), _ld(out_b), ptr(part), stream()))
    return out_a, out_b, part


def dwcat_reduce(part_u, part_i, d: int, heads: int, dwcat):
    _lib.check(_lib_().mmssl_dwcat_reduce(ptr(part_u), part_u.shape[0], ptr(part_i), part_i.shape[0], d, heads, ptr(dwcat), stream()))
    return dwcat


def combine_fwd(s, a, b, inv_layers: float, rate: float, out, want_sumsq: bool = True):
    lib = _lib_()
    n, d = s.shape
    npart = lib.mmssl_combine_partials(n, d)
    part = torch.empty(max(npart, 1), dtype=torch.float32, device=s.device) if want_sumsq else None
    _lib.check(lib.mmssl_combine_fwd(ptr(s), _ld(s), ptr(a), _ld(a), ptr(b), _ld(b), n, d, float(inv_layers), float(rate),
                                     ptr(out), _ld(out), ptr(part), npart, stream()))
    return out, (part[:npart] if part is not None else None)


def combine_bwd(g, a, b, ga_ext, gb_ext, rate: float, reg_coef: float, ga, gb):
    lib = _lib_()
    n, d = g.shape
    _lib.check(lib.mmssl_combine_bwd(ptr(g), _ld(g), ptr(a), _ld(a), ptr(b), _ld(b), ptr(ga_ext), _ld(ga_ext), ptr(gb_ext),
                                     _ld(gb_ext), n, d, float(rate), float(reg_coef), ptr(ga), _ld(ga), ptr(gb), _ld(gb), stream()))
    return ga, gb


def softmax_bwd(y, g, alpha: float, out):
    lib = _lib_()
    n, d = y.shape
    _lib.check(lib.mmssl_softmax_bwd(ptr(y), _ld(y), ptr(g), _ld(g), n, d, float(alpha), ptr(out), _ld(out), stream()))
    return out


def unit_rows(x, out=None):
    """out = x / max(|x|, 1e-12) row by row (F.normalize); a row's bits depend on that row only."""
    lib = _lib_()
    n, d = x.shape
    if out is None:
        out = torch.empty(n, d, dtype=torch.float32, device=x.device)
    _lib.check(lib.mmssl_unit_rows(ptr(x), _ld(x), n, d, ptr(out), _ld(out), stream()))
    return out


def axpby(x, alpha: float, beta: float, y, alpha_dev=None):
    lib = _lib_()
    n, d = x.shape
    _lib.check(lib.mmssl_axpby(ptr(x), _ld(x), n, d, float(alpha), ptr(alpha_dev), float(beta), ptr(y), _ld(y), stream()))
    return y


def mul_mask(x, mask, y):
    lib = _lib_()
    n, d = x.shape
    _lib.check(lib.mmssl_mul_mask(ptr(x), _ld(x), ptr(mask), _ld(mask), n, d, ptr(y), _ld(y), stream()))
    return y


def sumsq_partials(x):
    lib = _lib_()
    n, d = x.shape
    nb = lib.mmssl_sumsq_blocks(n, d)
    part = torch.empty(max(nb, 1), dtype=torch.float32, device=x.device)
    _lib.check(lib.mmssl_sumsq(ptr(x), _ld(x), n, d, ptr(part), stream()))
    return part[:nb]


def colsum(g, mask, out, accumulate=False):
    lib = _lib_()
    rows, n = g.shape
    _lib.check(lib.mmssl_colsum(ptr(g), _ld(g), ptr(mask), _ld(mask), rows, n, ptr(out), int(accumulate), stream()))
    return out


def bpr(uf, pf, nf, users, pos, neg, *, mode: int, reg_coef: float, g_mf=None, g_emb=None, part=None,
        g_u=None, g_p=None, g_n=None):
    """mmssl_bpr.  users/pos/neg: int64 device index tensors or None (identity)."""
    lib = _lib_()
    d = uf.shape[1]
    batch = int(users.numel()) if users is not None else uf.shape[0]
    nb = lib.mmssl_bpr_blocks(batch, d)
    if (mode & 1) and part is None:
        part = torch.empty(2 * max(nb, 1), dtype=torch.float32, device=uf.device)
    _lib.check(lib.mmssl_bpr(ptr(uf), _ld(uf), ptr(pf), _ld(pf), ptr(nf), _ld(nf), ptr(users), ptr(pos), ptr(neg), batch, d,
                             mode, float(reg_coef), ptr(g_mf), ptr(g_emb), ptr(part), ptr(g_u), _ld(g_u), ptr(g_p), _ld(g_p),
                             ptr(g_n), _ld(g_n), stream()))
    return part, nb


NCE_STREAMS = True      # tensor-core backward: its three products on three streams
NCE_IMPL = "auto"       # "auto": tensor cores where mmssl_infonce_tc_supported (n <= 2048, d in {64, 128}); "simt": CUDA cores


class InfoNCEWork:
    """Caller-owned work buffers of one InfoNCE evaluation (n rows, width d)."""

    def __init__(self, n: int, d: int, device, impl: Optional[str] = None):
        lib = _lib_()
        impl = NCE_IMPL if impl is None else impl
        self.tc = impl != "simt" and n > 0 and bool(lib.mmssl_infonce_tc_supported(n, d))
        self.ws = None
        if self.tc:      # exponentials (bf16 hi/lo), transposed operands and K-slice partials of the tensor-core path
            self.ws = torch.empty(lib.mmssl_infonce_tc_workspace_bytes(n, d), dtype=torch.uint8, device=device)
        f = dict(dtype=torch.float32, device=device)
        self.n, self.d = n, d
        self.a = torch.empty(n, d, **f); self.b = torch.empty(n, d, **f)
        self.na = torch.empty(n, **f); self.nb = torch.empty(n, **f)
        self.ga = torch.empty(n, d, **f); self.gb = torch.empty(n, d, **f)
        self.stats = torch.empty(lib.mmssl_infonce_stats_floats(n), **f)
        self.coef = torch.empty(2 * n, **f)
        self.n_loss_blocks = lib.mmssl_infonce_loss_blocks(n)
        self.loss_part = torch.empty(max(self.n_loss_blocks, 1), **f)


def infonce_forward(z1, z2, idx, inv_tau: float, work: InfoNCEWork, g_loss=None):
    """prepare + stats: fills work.loss_part (sum = n * loss) and the backward coefficients."""
    lib = _lib_()
    n, d = work.n, work.d
    if work.tc:      # gather + normalise + bf16 hi/lo split in one kernel, similarity tiles on wgmma, finalize
        _lib.check(lib.mmssl_infonce_forward_tc(ptr(z1), _ld(z1), ptr(z2), _ld(z2), ptr(idx), n, d, float(inv_tau), ptr(work.a), ptr(work.b),
                                                ptr(work.na), ptr(work.nb), ptr(work.stats), ptr(work.coef), ptr(g_loss),
                                                ptr(work.loss_part), ptr(work.ws), work.ws.numel(), stream()))
        return work.loss_part[:work.n_loss_blocks]
    _lib.check(lib.mmssl_infonce_prepare(ptr(z1), _ld(z1), ptr(z2), _ld(z2), ptr(idx), n, d, ptr(work.a), ptr(work.b),
                                         ptr(work.na), ptr(work.nb), ptr(work.ga), ptr(work.gb), stream()))
    _lib.check(lib.mmssl_infonce_stats(ptr(work.a), ptr(work.b), n, d, float(inv_tau), ptr(work.stats), ptr(work.coef),
                                       ptr(g_loss), ptr(work.loss_part), stream()))
    return work.loss_part[:work.n_loss_blocks]


def infonce_backward(idx, inv_tau: float, work: InfoNCEWork, g_z1, g_z2):
    """grad + scatter: accumulates d loss / d z1, z2 into g_z1 / g_z2 (tables when idx is given)."""
    lib = _lib_()
    n, d = work.n, work.d
    if work.tc:
        def phase(p):
            _lib.check(lib.mmssl_infonce_grad_tc(ptr(work.a), ptr(work.b), n, d, float(inv_tau), ptr(work.coef), ptr(work.stats),
                                                 ptr(work.ga), ptr(work.gb), ptr(work.ws), work.ws.numel(), p, stream()))
        if NCE_STREAMS:
            # the three products are independent: two of them on branches of their own (graph-capturable)
            from .engine import branch, join        # engine imports this module
            dev = work.a.device
            phase(0)
            with branch(dev, "nce2") as s2:
                phase(2)
            with branch(dev, "nce3") as s3:
                phase(3)
            phase(1)
            join(dev, s2, s3)
            phase(4)
        else:
            phase(-1)
    else:
        _lib.check(lib.mmssl_infonce_grad(ptr(work.a), ptr(work.b), n, d, float(inv_tau), ptr(work.coef), ptr(work.ga), ptr(work.gb), stream()))
    _lib.check(lib.mmssl_infonce_scatter(ptr(work.ga), ptr(work.gb), ptr(work.a), ptr(work.b), ptr(work.na), ptr(work.nb),
                                         ptr(idx), n, d, ptr(g_z1), _ld(g_z1), ptr(g_z2), _ld(g_z2), stream()))


def loss_assemble(bpr_part, n_bpr, batch, reg_coef, fr_u, fr_i, feat_coef, nce1, nce2, n_nce_rows, cl_rate, out5):
    lib = _lib_()
    _lib.check(lib.mmssl_loss_assemble(ptr(bpr_part), n_bpr, batch, float(reg_coef), ptr(fr_u),
                                       0 if fr_u is None else fr_u.numel(), ptr(fr_i), 0 if fr_i is None else fr_i.numel(),
                                       float(feat_coef), ptr(nce1), 0 if nce1 is None else nce1.numel(), ptr(nce2),
                                       0 if nce2 is None else nce2.numel(), n_nce_rows, float(cl_rate), ptr(out5), stream()))
    return out5


def step_tick(step_dev):
    _lib.check(_lib_().mmssl_step_tick(ptr(step_dev), stream()))


def adamw(params, grads, ms, vs, step_dev, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2):
    lib = _lib_()
    for lo in range(0, len(params), 16):
        p = params[lo:lo + 16]; g = grads[lo:lo + 16]; m = ms[lo:lo + 16]; v = vs[lo:lo + 16]
        n = len(p)
        arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
        numel = (C.c_int64 * n)(*[t.numel() for t in p])
        for t in (*p, *g, *m, *v):
            assert t.is_contiguous() and t.dtype == torch.float32
        _lib.check(lib.mmssl_adamw(n, arr(p), arr(g), arr(m), arr(v), numel, ptr(step_dev), float(lr), float(beta1),
                                   float(beta2), float(eps), float(weight_decay), stream()))


# ---- projection pieces -----------------------------------------------------------------------
def proj_epilogue(partial, split_k, m, n, bias, mask, y, y_pre=None):
    lib = _lib_()
    _lib.check(lib.mmssl_proj_epilogue(ptr(partial), split_k, m, n, ptr(bias), ptr(mask), _ld(mask), ptr(y), _ld(y),
                                       ptr(y_pre), _ld(y_pre), stream()))
    return y


def wgrad_epilogue(partial, split_k, m, n, dw, accumulate=False):
    lib = _lib_()
    _lib.check(lib.mmssl_wgrad_epilogue(ptr(partial), split_k, m, n, ptr(dw), dw.stride(0), int(accumulate), stream()))
    return dw


def split_bf16(x, ldo=None, out=None):
    """fp32 [rows, cols] -> (hi, lo) bf16 [rows, ldo] with zero padding (ldo % 8 == 0 for TMA strides)."""
    lib = _lib_()
    rows, cols = x.shape
    if ldo is None:
        ldo = (cols + 7) // 8 * 8
    if out is None:
        hi = torch.empty(rows, ldo, dtype=torch.bfloat16, device=x.device)
        lo = torch.empty(rows, ldo, dtype=torch.bfloat16, device=x.device)
    else:
        hi, lo = out
    _lib.check(lib.mmssl_split_bf16(ptr(x), x.stride(0), rows, cols, ptr(hi), ptr(lo), ldo, stream()))
    return hi, lo


def split_bf16_t(x, mask=None, ldo=None, out=None, colsum=None):
    """fp32 [rows, cols] (optionally * mask) -> transposed (hi, lo) bf16 [cols, ldo], zero padded.
    colsum: optional fp32 [cols] that receives the column sums of (x * mask) from the same pass."""
    lib = _lib_()
    rows, cols = x.shape
    if ldo is None:
        ldo = (rows + 7) // 8 * 8
    if out is None:
        hi = torch.empty(cols, ldo, dtype=torch.bfloat16, device=x.device)
        lo = torch.empty(cols, ldo, dtype=torch.bfloat16, device=x.device)
    else:
        hi, lo = out
    if colsum is not None:
        assert colsum.dtype == torch.float32 and colsum.numel() == cols and colsum.is_contiguous()
        _lib.check(lib.mmssl_split_bf16_t_colsum(ptr(x), x.stride(0), ptr(mask), _ld(mask), rows, cols, ptr(hi), ptr(lo), ldo,
                                                 ptr(colsum), stream()))
    else:
        _lib.check(lib.mmssl_split_bf16_t(ptr(x), x.stride(0), ptr(mask), _ld(mask), rows, cols, ptr(hi), ptr(lo), ldo, stream()))
    return hi, lo


def gemm_bf16x3_wide(a_hi, a_lo, b_hi, b_lo, m, n, k, out, alpha: float = 1.0, accumulate: bool = False):
    """out[m, n] (+)= alpha * (a_hi + a_lo)[m,k] @ (b_hi + b_lo)[n,k]^T on wgmma tensor cores, any n (csrc/gemm_wide.cu)."""
    lib = _lib_()
    assert out.dtype == torch.float32 and out.stride(1) == 1 and out.shape == (m, n)
    _lib.check(lib.mmssl_gemm_bf16x3_wide(ptr(a_hi), ptr(a_lo), a_hi.stride(0), ptr(b_hi), ptr(b_lo), b_hi.stride(0), m, n, k,
                                          float(alpha), int(accumulate), ptr(out), out.stride(0), stream()))
    return out


def gemm_wide_set_chunk(k_blocks: int) -> None:
    """k-blocks (64 of K) accumulated in registers before a pass is folded into C in fp32 (default 16; csrc/gemm_wide.cu)."""
    _lib.check(_lib_().mmssl_gemm_wide_set_chunk(int(k_blocks)))


def spmm_plan_set_cuts(split_threshold: int, seg_len: int, heavy_threshold: int = 1024, heavy_seg_len: int = 64) -> None:
    """Where the SpMM work plan cuts rows (csrc/graph.cu); applies to graphs built afterwards."""
    _lib.check(_lib_().mmssl_spmm_plan_set_cuts(int(split_threshold), int(seg_len), int(heavy_threshold), int(heavy_seg_len)))


def spmm_pipe_set_blocks(blocks: int) -> None:
    """Grid size (blocks of 128 threads) of the software-pipelined SpMM (impl bit SPMM_IMPL_PIPE); 0 = one resident wave."""
    _lib.check(_lib_().mmssl_spmm_pipe_set_blocks(int(blocks)))


def gemm_bf16x3_plan(m, n, k):
    lib = _lib_()
    sk = C.c_int(0)
    floats = lib.mmssl_gemm_bf16x3_workspace_floats(m, n, k, C.byref(sk))
    return int(floats), int(sk.value)


def gemm_bf16x3(a_hi, a_lo, b_hi, b_lo, m, n, k, split_k, partial):
    """partial[s][m][n] = K-slice s of (a_hi + a_lo)[m,k] @ (b_hi + b_lo)[n,k]^T on wgmma tensor cores."""
    lib = _lib_()
    _lib.check(lib.mmssl_gemm_bf16x3(ptr(a_hi), ptr(a_lo), a_hi.stride(0), ptr(b_hi), ptr(b_lo), b_hi.stride(0), m, n, k,
                                     split_k, ptr(partial), stream()))
    return partial


def gemm_bf16x3_group_plan(shapes, max_ctas=0, units=False):
    """Plan of one grouped launch over 1-2 problems, shapes = [(m, n, k), ...] with the same n.
    Returns (splits, floats) per problem; with units=True also the [n_units, 4] int32 list (problem, m_tile, kb_begin,
    kb_end) in the order the CTAs walk it."""
    lib = _lib_()
    np_ = len(shapes)
    mnk = (C.c_int64 * (3 * np_))(*[int(v) for s in shapes for v in s])
    sk = (C.c_int32 * np_)()
    fl = (C.c_int64 * np_)()
    n_units = lib.mmssl_gemm_bf16x3_group_plan(np_, mnk, int(max_ctas), sk, fl, None, 0)
    if n_units < 0:
        _lib.check(1)
    splits, floats = [int(v) for v in sk], [int(v) for v in fl]
    if not units:
        return splits, floats
    buf = torch.zeros(n_units, 4, dtype=torch.int32, device="cpu")
    lib.mmssl_gemm_bf16x3_group_plan(np_, mnk, int(max_ctas), sk, fl, C.c_void_p(buf.data_ptr()), n_units)
    return splits, floats, buf


def gemm_bf16x3_group(problems, max_ctas=0):
    """One persistent launch for 1-2 problems (a_hi, a_lo, b_hi, b_lo, m, n, k, split_k, partial): each partial[s][m][n]
    as gemm_bf16x3 with the same split_k computes it."""
    lib = _lib_()
    arr = (_lib.GemmProblem * len(problems))()
    for q, (a_hi, a_lo, b_hi, b_lo, m, n, k, sk, part) in zip(arr, problems):
        q.a_hi, q.a_lo, q.lda = a_hi.data_ptr(), a_lo.data_ptr(), a_hi.stride(0)
        q.b_hi, q.b_lo, q.ldb = b_hi.data_ptr(), b_lo.data_ptr(), b_hi.stride(0)
        q.m, q.n, q.k, q.split_k, q.partial = m, n, k, sk, part.data_ptr()
    _lib.check(lib.mmssl_gemm_bf16x3_group(len(problems), arr, int(max_ctas), stream()))
