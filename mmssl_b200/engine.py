"""Forward / backward schedule of the MMSSL hot path on the CUDA library.

Implements the closed form of ``MMSSL.forward`` (reference Models.py:171-220; SURVEY.md appendix A)
and its hand-derived backward as an explicit sequence of library kernels.  No autograd inside:
``functional.MMSSLForwardFn`` wraps it for the drop-in ``Models.MMSSL`` and ``hotstep.HotStep``
drives it directly (fused with the loss kernels and AdamW, CUDA-graph captured).

Launch inventory of one forward (K GCN layers, modality graphs aliasing ui/iu as at step 0,
main.py:68-69):  2 W splits + 1 grouped projection GEMM + 2 epilogues + 2 two-RHS SpMM (image|text batched)
+ 2 id SpMM + Wsum + 2 fused id-fusion kernels + 2K SpMM (softmax / layer-sum fused) + 2 combine kernels,
scheduled on three streams (see ``Engine.two_streams``).
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib, ops
from .graph import BipartiteGraph

P_WV, P_BV, P_WT, P_BT = "image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias"
P_EU, P_EI, P_WCAT = "user_id_embedding.weight", "item_id_embedding.weight", "weight_dict.w_self_attention_cat"
LIVE = (P_WV, P_BV, P_WT, P_BT, P_EU, P_EI, P_WCAT)
SUPPORTED_WIDTHS = (32, 64, 96, 128, 192, 256)   # for messages; the library's mmssl_embed_width_supported decides


class FeatureStore:
    """Constant modality features (Models.py:46-47) prepared once for the tensor-core projection:
    bf16 hi/lo split of F [I, D] (forward operand) and of F^T [D, I] (weight-gradient operand)."""

    def __init__(self, feats: torch.Tensor, keep_fp32: bool = True):
        assert feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 2
        self.n_items, self.dim = feats.shape
        self.hi, self.lo = ops.split_bf16(feats)            # [I, ceil8(D)]
        self.t_hi, self.t_lo = ops.split_bf16_t(feats)      # [D, ceil8(I)]
        self.fp32 = feats if keep_fp32 else None

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in (self.hi, self.lo, self.t_hi, self.t_lo))


@dataclass
class FwdState:
    graphs: tuple
    masks: Optional[tuple]
    X2: torch.Tensor
    U2: torch.Tensor
    I2: torch.Tensor
    id_out: tuple                      # (Uvid, Utid, Ivid, Itid)
    fused: bool
    wsum: Optional[torch.Tensor] = None
    wsum_t: Optional[torch.Tensor] = None
    zn_u: Optional[torch.Tensor] = None
    nrm_u: Optional[torch.Tensor] = None
    zn_i: Optional[torch.Tensor] = None
    nrm_i: Optional[torch.Tensor] = None
    u_last: Optional[torch.Tensor] = None   # softmax outputs of the last GCN layer
    i_last: Optional[torch.Tensor] = None
    sumsq_u: Optional[torch.Tensor] = None  # per-block sum(Uv^2+Ut^2) / (Iv^2+It^2) for feat_reg
    sumsq_i: Optional[torch.Tensor] = None
    u0: Optional[torch.Tensor] = None       # keep_fold: the user id rows after the id fusion (u_0) ...
    i_layers: Optional[tuple] = None        # ... and the item layer tables i_0 .. i_{K-1} the user layers gather (foldin.py)


# The branches of the step and the priority of each one's stream (0 = lowest .. -5): the item-side twin of the critical id / GCN
# chain ("pair") and the two side products of the tensor-core InfoNCE backward run ahead of the projection branch ("side").
PRIORITY = {"side": 0, "pair": -1, "fork2": 0, "fork3": 0, "pre": 0, "loss": 0, "nce2": -1, "nce3": -1}
_streams: Dict[Tuple, torch.cuda.Stream] = {}


@contextlib.contextmanager
def branch(dev, name: str, on: bool = True):
    """Fork branch `name` of the step: the body is issued on that branch's stream (one per device and name), after the work
    issued so far on the current stream.  Yields the stream for `join`, which the caller places where the branch's results are
    needed.  With `on` False the body runs on the current stream and None is yielded."""
    if not on:
        yield None
        return
    key = (dev.type, dev.index, name)
    st = _streams.get(key)
    if st is None:
        st = _streams[key] = torch.cuda.Stream(device=dev, priority=PRIORITY[name])
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        yield st


def join(dev, *branches) -> None:
    """The current stream waits for the work issued so far on `branches` (None stands for a branch that ran inline)."""
    cur = torch.cuda.current_stream(dev)
    for st in branches:
        if st is not None:
            cur.wait_stream(st)


def capture_graph(warmup, body):
    """Runs `warmup` on a stream forked from the current one (so that every lazily created buffer and stream exists), waits for
    the device, then captures `body` into a CUDA graph.  Returns (graph, what `body` returned)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        warmup()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = body()
    return g, out


class Engine:
    def __init__(self, embed_size: int, n_layers: int, head_num: int = 4, id_cat_rate: float = 0.36,
                 model_cat_rate: float = 0.55, proj_impl: str = "tc"):
        if not _lib.load().mmssl_embed_width_supported(int(embed_size)):
            raise ValueError(f"embed_size {embed_size} is not supported: mmssl_b200 kernels are built for {SUPPORTED_WIDTHS}")
        self.d, self.K, self.H = embed_size, n_layers, head_num
        self.id_rate, self.cat_rate = id_cat_rate, model_cat_rate
        self.proj_impl = proj_impl
        # Grid of the grouped projection GEMM: one CTA per SM (132 on the H100 SXM) rather than the full two-per-SM wave.  The
        # persistent CTAs would otherwise hold every slot while the id / GCN branch runs beside them; measured on an H100 at
        # 700 W, 132 CTAs gave the shorter Baby and Sports steps (DESIGN section 6).
        self.proj_max_ctas = 132
        self._tile_id: Dict[Tuple, torch.Tensor] = {}
        # The modality branch (projection -> A_ui [Xv|Xt] -> A_iu [Uv|Ut]) and the id/GCN branch are
        # independent until the final combine (and again after combine-backward), so they run on two
        # streams; inside a CUDA graph they become parallel branches.  Set to False to serialise.
        self.two_streams = True
        # Row-sharded scheme (SURVEY 8e, rowshard_step.py): every table is a row block, the graphs are row blocks with
        # global column ids, and each SpMM needs its dense operand from all ranks.  ``exchange(list_of_local, space)``
        # ('u' = user rows, 'i' = item rows) returns the gathered operands; None = single GPU, operands pass through.
        self.exchange = None
        self.sharded_spmm = None            # callable(g, which, xs, space, ys, **spmm_kwargs) -> list of local outputs

    def _full(self, xs, space: str):
        return xs if self.exchange is None else self.exchange(xs, space)

    def _spmm(self, g, which: str, xs, space: str, ys=None, **kw):
        """One propagation product  Y = epi(op(g) @ X):  which = 'fwd' (A) or 'bwd' (A^T); `space` names the row space the dense
        operand lives in ('u' users / 'i' items).  Single GPU: the operand passes through.  Row-sharded: `sharded_spmm`
        (rowshard_step.py) decides how the operand / the result crosses the GPUs (all-gather of the operand, or partial products
        + reduce-scatter of the result, whichever moves the item-sized table)."""
        if self.sharded_spmm is not None:
            return self.sharded_spmm(g, which, xs, space, ys, **kw)
        return ops.spmm(getattr(g, which), self._full(xs, space), ys, **kw)

    def branch(self, dev, name: str, on: bool = True):
        """`branch` of this engine's schedule: inline when `two_streams` is off."""
        return branch(dev, name, on and self.two_streams)

    def _fork(self, dev, name: str, fn_a, fn_b):
        """Two independent kernel groups: fn_a on the current stream, fn_b beside it on branch `name`, joined at once (a, then b,
        on one stream when `two_streams` is off).  Returns (fn_a(), fn_b())."""
        if not self.two_streams:
            return fn_a(), fn_b()
        with branch(dev, name) as st:
            rb = fn_b()
        ra = fn_a()
        join(dev, st)
        return ra, rb

    # ------------------------------------------------------------------ helpers
    def _tile(self, dev) -> torch.Tensor:
        """[d, H*d] = H identities side by side:  Wsum = T @ Wcat,  dWcat = T^T @ dWsum."""
        key = (dev.type, dev.index)
        t = self._tile_id.get(key)
        if t is None:
            t = torch.eye(self.d, device=dev, dtype=torch.float32).repeat(1, self.H).contiguous()
            self._tile_id[key] = t
        return t

    def _new(self, *shape, dev):
        return torch.empty(*shape, dtype=torch.float32, device=dev)

    # ------------------------------------------------------------------ projection
    def _project(self, P, feats, masks, ys, wait_for=None, plan_rows=None):
        """X = F W^T + b, then the dropout mask, for image and text (Models.py:173-174).  Tensor cores: both GEMMs in ONE
        grouped persistent launch (the feature streams of 118 + 30 MB at Baby share one balanced wave), then the two
        split-K epilogues.  `wait_for`: a branch whose work (the mask draws) the epilogues wait for; the GEMM does not.
        `plan_rows`: the row count the K split is planned for (default: the rows projected).  The split fixes the order in which
        a row's products are summed, so rows projected in launches of different heights under one plan_rows get the same
        bits: a rank's item block, or a few feature rows, projects as the whole catalogue does (similar.py)."""
        d = self.d
        dev = ys[0].device
        ws, bs = (P[P_WV], P[P_WT]), (P[P_BV], P[P_BT])
        if self.proj_impl != "tc":
            join(dev, wait_for)
            self._fork(dev, "fork2", lambda: self._project_simt(ws[0], bs[0], feats[0], masks[0], ys[0]),
                       lambda: self._project_simt(ws[1], bs[1], feats[1], masks[1], ys[1]))
            return
        if plan_rows is None:
            splits, floats = ops.gemm_bf16x3_group_plan([(fs.n_items, d, fs.dim) for fs in feats], self.proj_max_ctas)
        else:
            splits, _ = ops.gemm_bf16x3_group_plan([(int(plan_rows), d, fs.dim) for fs in feats], self.proj_max_ctas)
            floats = [sk * fs.n_items * d for sk, fs in zip(splits, feats)]
        parts = self._new(sum(floats), dev=dev).split(floats)
        probs = []
        for w, fs, sk, part in zip(ws, feats, splits, parts):
            w_hi, w_lo = ops.split_bf16(w)
            probs.append((fs.hi, fs.lo, w_hi, w_lo, fs.n_items, d, fs.dim, sk, part))
        ops.gemm_bf16x3_group(probs, self.proj_max_ctas)
        join(dev, wait_for)
        for b, fs, sk, part, mask, y in zip(bs, feats, splits, parts, masks, ys):
            ops.proj_epilogue(part, sk, fs.n_items, d, b, mask, y)

    def _project_simt(self, w, b, fs: FeatureStore, mask, y):
        I, d = fs.n_items, self.d
        if fs.fp32 is None:
            raise RuntimeError("proj_impl='simt' needs the fp32 features (keep_fp32=True)")
        part = self._new(I, d, dev=y.device)
        ops.sgemm(fs.fp32, w, part, trans_b=True)
        ops.proj_epilogue(part, 1, I, d, b, mask, y)

    def _project_bwd(self, gxs, masks, feats, dws, dbs):
        """dW[d,D] = (gx*mask)^T F ; db = colsum(gx*mask), for image and text.  Tensor cores: the operand splits (db from
        the same pass), both weight-gradient GEMMs in ONE grouped persistent launch, then the two epilogues."""
        d = self.d
        if self.proj_impl != "tc":
            self._fork(gxs[0].device, "fork2", lambda: self._project_bwd_simt(gxs[0], masks[0], feats[0], dws[0], dbs[0]),
                       lambda: self._project_bwd_simt(gxs[1], masks[1], feats[1], dws[1], dbs[1]))
            return
        splits, floats = ops.gemm_bf16x3_group_plan([(fs.dim, d, fs.n_items) for fs in feats], self.proj_max_ctas)
        parts = self._new(sum(floats), dev=gxs[0].device).split(floats)
        probs = []
        for gx, mask, fs, db, sk, part in zip(gxs, masks, feats, dbs, splits, parts):
            g_hi, g_lo = ops.split_bf16_t(gx, mask, ldo=fs.t_hi.shape[1], colsum=db)   # [d, ceil8(I)]
            probs.append((fs.t_hi, fs.t_lo, g_hi, g_lo, fs.dim, d, fs.n_items, sk, part))
        ops.gemm_bf16x3_group(probs, self.proj_max_ctas)
        for fs, sk, part, dw in zip(feats, splits, parts, dws):
            ops.wgrad_epilogue(part, sk, fs.dim, d, dw)

    def _project_bwd_simt(self, gx, mask, fs: FeatureStore, dw, db):
        I, d = fs.n_items, self.d
        gm = self._new(I, d, dev=gx.device)
        ops.mul_mask(gx, mask, gm)
        ops.sgemm(gm, fs.fp32, dw, trans_a=True)
        ops.colsum(gx, mask, db)

    # ------------------------------------------------------------------ forward
    def forward(self, P: Dict[str, torch.Tensor], feats: Tuple[FeatureStore, FeatureStore],
                graphs: Sequence[BipartiteGraph], masks, want_sumsq: bool = True, side_pre=None, keep_fold: bool = False):
        """masks: None, a pair of [I, d] keep-masks (0 or 1/(1-p)), or a callable returning one -- the
        callable and `side_pre` run on a branch forked at the head of the modality branch, i.e. off the critical path: the
        projection GEMM starts at once, and only its epilogues (which apply the masks) wait for that branch.
        keep_fold: the returned state also holds u_0 and the item layer tables i_0 .. i_{K-1} (references to tables the forward
        computes anyway: the same kernels and launches), which with X2 are what a user row is folded from (foldin.py)."""
        g_ui, g_iu, g_vui, g_viu, g_tui, g_tiu = graphs
        U, I = g_ui.shape
        d, K = self.d, self.K
        e_u, e_i = P[P_EU], P[P_EI]
        dev = e_u.device
        X2, U2, I2 = self._new(I, 2 * d, dev=dev), self._new(U, 2 * d, dev=dev), self._new(I, 2 * d, dev=dev)
        xv, xt = X2[:, :d], X2[:, d:]
        uv, ut = U2[:, :d], U2[:, d:]
        iv, it = I2[:, :d], I2[:, d:]

        with self.branch(dev, "side") as side:                                      # the modality branch
            with self.branch(dev, "pre", on=side_pre is not None or callable(masks)) as pre:
                if side_pre is not None:
                    side_pre()
                m = masks() if callable(masks) else masks
            # the modality branch joins the main stream before the loss kernels, so `pre` (seed memset, sampler) is joined too
            self._project(P, feats, m if m else (None, None), (xv, xt), wait_for=pre)   # Models.py:173-174
            self._spmm(g_ui, "fwd", [xv, xt], "i", [uv, ut])                        # :177,182
            self._spmm(g_iu, "fwd", [uv, ut], "u", [iv, it])                        # :178,183

        def id_prop(ga, gb, e, rows, space):                                           # :179-180,185-186
            def one(g):
                if g.nnz == 0:
                    return torch.zeros(rows, d, dtype=torch.float32, device=dev)
                return self._spmm(g, "fwd", [e], space)[0]
            ya = one(ga)
            return (ya, ya) if ga is gb else (ya, one(gb))

        (uvid, utid), (ivid, itid) = self._fork(dev, "pair", lambda: id_prop(g_vui, g_tui, e_i, U, "i"),
                                                lambda: id_prop(g_viu, g_tiu, e_u, I, "u"))
        st = FwdState(tuple(graphs), m, X2, U2, I2, (uvid, utid, ivid, itid),
                      fused=any(g.nnz > 0 for g in (g_vui, g_viu, g_tui, g_tiu)))
        if st.fused:                                                                   # :188-197 (closed form)
            if d in (64, 128):      # fused row x matrix kernels, Wsum in shared memory
                st.wsum, st.wsum_t = ops.wsum(P[P_WCAT], d, self.H)

                def fuse(ya, yb, e):
                    return ops.id_fuse2_fwd(ya, None if ya is yb else yb, 1.0 if ya is yb else 0.5, st.wsum, e, self.id_rate)
            else:                   # d = 32, 96, 192, 256: no fused kernel at these widths (the d x d matrix of 256 does not fit
                                    # shared memory) -> GEMM path
                st.wsum = ops.sgemm(self._tile(dev), P[P_WCAT], self._new(d, d, dev=dev))

                def fuse(ya, yb, e):
                    z = self._new(e.shape[0], d, dev=dev)
                    if ya is yb:
                        ops.sgemm(ya, st.wsum, z)
                    else:
                        ops.sgemm(ya, st.wsum, z, alpha=0.5)
                        ops.sgemm(yb, st.wsum, z, alpha=0.5, beta=1.0)
                    out = self._new(e.shape[0], d, dev=dev)
                    return ops.id_fuse_fwd(z, e, self.id_rate, out)

            (u0, st.zn_u, st.nrm_u), (i0, st.zn_i, st.nrm_i) = self._fork(dev, "pair", lambda: fuse(uvid, utid, e_u),
                                                                          lambda: fuse(ivid, itid, e_i))
        else:
            u0, i0 = e_u, e_i
        # GCN layers: u_{k+1} = A_ui i_k ; i_{k+1} = A_iu u_{k+1}; softmax on the last one (:201-211);
        # the layer sums S_u, S_i accumulate in the SpMM epilogue (:213-214)
        s_u, s_i = self._new(U, d, dev=dev), self._new(I, d, dev=dev)
        cur_i = i0
        if keep_fold:
            st.u0, st.i_layers = u0, ()
        if K == 0:
            ops.axpby(u0, 1.0, 0.0, s_u)
            ops.axpby(i0, 1.0, 0.0, s_i)
        for k in range(K):
            last = k == K - 1
            epi = ops.EPI_SOFTMAX if last else ops.EPI_NONE
            mode = 2 if k == 0 else 1
            if keep_fold:
                st.i_layers += (cur_i,)
            u_n = self._spmm(g_ui, "fwd", [cur_i], "i", epilogue=epi, ss=[s_u], s_mode=mode, sbases=[u0] if k == 0 else None)[0]
            i_n = self._spmm(g_iu, "fwd", [u_n], "u", epilogue=epi, ss=[s_i], s_mode=mode, sbases=[i0] if k == 0 else None)[0]
            if last:
                st.u_last, st.i_last = u_n, i_n
            cur_i = i_n
        inv = 1.0 / (K + 1)
        join(dev, side)                 # the combine needs Uv|Ut and Iv|It
        (u_f, st.sumsq_u), (i_f, st.sumsq_i) = self._fork(
            dev, "pair", lambda: ops.combine_fwd(s_u, uv, ut, inv, self.cat_rate, self._new(U, d, dev=dev), want_sumsq),      # :213,217
            lambda: ops.combine_fwd(s_i, iv, it, inv, self.cat_rate, self._new(I, d, dev=dev), want_sumsq))          # :214,218
        outs = (u_f, i_f, iv, it, uv, ut, uvid, utid, ivid, itid)
        return outs, st

    # ------------------------------------------------------------------ backward
    def backward(self, st: FwdState, P: Dict[str, torch.Tensor], feats, grads: Sequence[Optional[torch.Tensor]],
                 feat_reg_coef: float = 0.0, out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """grads: d loss / d (u_f, i_f, Iv, It, Uv, Ut, Uvid, Utid, Ivid, Itid), entries may be None.
        feat_reg_coef folds d(feat_reg)/d(Uv,Ut,Iv,It) = coef * x into the combine-backward kernel.
        Returns gradients for the live parameters (written into `out` when given)."""
        g_ui, g_iu, g_vui, g_viu, g_tui, g_tiu = st.graphs
        U, I = g_ui.shape
        d, K = self.d, self.K
        dev = st.X2.device
        inv = 1.0 / (K + 1)

        def prep(g, rows):
            if g is None:
                return None
            if g.dtype != torch.float32 or g.stride(1) != 1 or g.stride(0) % 4 or g.data_ptr() % 16:
                g = g.contiguous().float()
            assert g.shape == (rows, d)
            return g

        g_uf, g_if = prep(grads[0], U), prep(grads[1], I)
        g_iv, g_it, g_uv, g_ut = prep(grads[2], I), prep(grads[3], I), prep(grads[4], U), prep(grads[5], U)
        g_uvid, g_utid, g_ivid, g_itid = prep(grads[6], U), prep(grads[7], U), prep(grads[8], I), prep(grads[9], I)
        if g_uf is None:
            g_uf = torch.zeros(U, d, dtype=torch.float32, device=dev)
        if g_if is None:
            g_if = torch.zeros(I, d, dtype=torch.float32, device=dev)
        res = out if out is not None else {}

        def slot(name, like):
            t = res.get(name)
            if t is None:
                t = torch.empty_like(like)
                res[name] = t
            return t

        uv, ut = st.U2[:, :d], st.U2[:, d:]
        iv, it = st.I2[:, :d], st.I2[:, d:]
        # ---- combine backward (Models.py:213-218): through the two normalisations (+ feat_reg)
        gU2, gI2 = self._new(U, 2 * d, dev=dev), self._new(I, 2 * d, dev=dev)
        self._fork(dev, "pair", lambda: ops.combine_bwd(g_uf, uv, ut, g_uv, g_ut, self.cat_rate, feat_reg_coef, gU2[:, :d], gU2[:, d:]),
                   lambda: ops.combine_bwd(g_if, iv, it, g_iv, g_it, self.cat_rate, feat_reg_coef, gI2[:, :d], gI2[:, d:]))
        w_slots = (slot(P_WV, P[P_WV]), slot(P_BV, P[P_BV]), slot(P_WT, P[P_WT]), slot(P_BT, P[P_BT]))

        with self.branch(dev, "side") as side:
            # modality propagation backward (Models.py:177-178,182-183), image|text batched, then the
            # projection backward (dropout mask folded into the operand split)
            self._spmm(g_iu, "bwd", [gI2[:, :d], gI2[:, d:]], "i", [gU2[:, :d], gU2[:, d:]], cs=[gU2[:, :d], gU2[:, d:]], alpha=1.0)
            gX2 = self._new(I, 2 * d, dev=dev)
            self._spmm(g_ui, "bwd", [gU2[:, :d], gU2[:, d:]], "u", [gX2[:, :d], gX2[:, d:]])
            m = st.masks
            self._project_bwd((gX2[:, :d], gX2[:, d:]), m if m else (None, None), feats, (w_slots[0], w_slots[2]),
                              (w_slots[1], w_slots[3]))
        # ---- GCN backward.  every u_k, i_k receives inv * g_uf / inv * g_if from the layer mean.
        # d loss / d u_0 = inv * g_uf (u_0 only feeds the layer mean): needed only after the chain -> issued first, on the pair stream
        g_eu = slot(P_EU, P[P_EU])
        g_ei = slot(P_EI, P[P_EI])

        def chain():
            if K == 0:
                return ops.axpby(g_if, inv, 0.0, g_ei)
            t = ops.softmax_bwd(st.i_last, g_if, inv, self._new(I, d, dev=dev))
            for k in range(K - 1, -1, -1):
                last = k == K - 1
                tu = self._spmm(g_iu, "bwd", [t], "i", cs=[g_uf], alpha=inv,
                                epilogue=ops.EPI_SOFTMAX_BWD if last else ops.EPI_NONE,
                                ysaved=[st.u_last] if last else None)[0]
                # the last product of the chain IS d loss / d i_0: it lands in the item table's gradient slot
                t = self._spmm(g_ui, "bwd", [tu], "u", [g_ei] if k == 0 else None, cs=[g_if], alpha=inv)[0]
            return t

        # ---- id fusion backward (Models.py:188-197)
        uvid, utid, ivid, itid = st.id_out
        g_wcat = slot(P_WCAT, P[P_WCAT])
        dwcat_args = None
        fused2 = st.fused and d in (64, 128)
        if fused2:
            def fuse_bwd2(g0, zn, nrm, ya, yb, g_ya, g_yb):
                same = ya is yb
                oa, ob, part = ops.id_fuse2_bwd(g0, zn, nrm, ya, None if same else yb, 1.0 if same else 0.5, st.wsum_t,
                                                self.id_rate, g_ya, g_yb, two_outputs=not same)
                return oa, (oa if same else ob), part

            # The user-side fusion backward needs only g_eu = inv * g_uf, not the chain: it runs beside the chain on the pair
            # stream (after the chain it had to share the SMs with the weight-gradient GEMMs' large CTAs and ran several times
            # slower on the earlier hardware); only the item side, which reads the chain's result g_ei, follows the chain.
            def user_side():
                ops.axpby(g_uf, inv, 0.0, g_eu)
                return fuse_bwd2(g_eu, st.zn_u, st.nrm_u, uvid, utid, g_uvid, g_utid)

            _, (gt_uvid, gt_utid, part_u) = self._fork(dev, "pair", chain, user_side)
            gt_ivid, gt_itid, part_i = fuse_bwd2(g_ei, st.zn_i, st.nrm_i, ivid, itid, g_ivid, g_itid)
            dwcat_args = (part_u, part_i)
        else:
            self._fork(dev, "pair", chain, lambda: ops.axpby(g_uf, inv, 0.0, g_eu))
        if not st.fused:
            g_wcat.zero_()
            gt_uvid, gt_utid, gt_ivid, gt_itid = g_uvid, g_utid, g_ivid, g_itid
        elif not fused2:
            d_wsum = torch.zeros(d, d, dtype=torch.float32, device=dev)

            def fuse_bwd(g0, zn, nrm, ya, yb, g_ya, g_yb, rows):
                dz = ops.id_fuse_bwd(g0, zn, nrm, self.id_rate, self._new(rows, d, dev=dev))
                sk = max(1, min(256, rows // 128))
                if ya is yb:
                    ops.sgemm(ya, dz, d_wsum, trans_a=True, alpha=1.0, beta=1.0, split_k=sk)
                    tot = self._new(rows, d, dev=dev)
                    ops.sgemm(dz, st.wsum, tot, trans_b=True)                    # dz @ Wsum^T
                    for g in (g_ya, g_yb):
                        if g is not None:
                            ops.axpby(g, 1.0, 1.0, tot)
                    return tot, tot
                ops.sgemm(ya, dz, d_wsum, trans_a=True, alpha=0.5, beta=1.0, split_k=sk)
                ops.sgemm(yb, dz, d_wsum, trans_a=True, alpha=0.5, beta=1.0, split_k=sk)
                ta = self._new(rows, d, dev=dev)
                ops.sgemm(dz, st.wsum, ta, trans_b=True, alpha=0.5)
                tb = ta
                if g_ya is not None or g_yb is not None:
                    tb = ta.clone()
                    if g_ya is not None:
                        ops.axpby(g_ya, 1.0, 1.0, ta)
                    if g_yb is not None:
                        ops.axpby(g_yb, 1.0, 1.0, tb)
                return ta, tb

            gt_uvid, gt_utid = fuse_bwd(g_eu, st.zn_u, st.nrm_u, uvid, utid, g_uvid, g_utid, U)
            gt_ivid, gt_itid = fuse_bwd(g_ei, st.zn_i, st.nrm_i, ivid, itid, g_ivid, g_itid, I)
            ops.sgemm(self._tile(dev), d_wsum, g_wcat, trans_a=True)            # dWcat[h] = dWsum for every head

        def id_prop_bwd(ga, gb, gya, gyb, g_e, same_out, space):
            # E-gradient += A^T g  for each modality graph (same_out: both modalities share graph and output)
            if ga is gb:
                if ga.nnz == 0:
                    return
                if same_out and gya is not None:
                    self._spmm(ga, "bwd", [gya], space, [g_e], cs=[g_e], alpha=1.0)
                    return
                for g in (gya, gyb):
                    if g is not None:
                        self._spmm(ga, "bwd", [g], space, [g_e], cs=[g_e], alpha=1.0)
                return
            for gr, g in ((ga, gya), (gb, gyb)):
                if g is not None and gr.nnz > 0:
                    self._spmm(gr, "bwd", [g], space, [g_e], cs=[g_e], alpha=1.0)

        # Uvid = A_vui E_i, Utid = A_tui E_i -> gradient flows to E_i; Ivid/Itid -> E_u.  The head reduction of dWcat feeds
        # nothing else of the step: it runs beside the two propagations on a third stream.
        def props():
            self._fork(dev, "pair", lambda: id_prop_bwd(g_vui, g_tui, gt_uvid, gt_utid, g_ei, st.fused and uvid is utid, "u"),
                       lambda: id_prop_bwd(g_viu, g_tiu, gt_ivid, gt_itid, g_eu, st.fused and ivid is itid, "i"))

        def head_reduce():
            if dwcat_args is not None:
                ops.dwcat_reduce(dwcat_args[0], dwcat_args[1], d, self.H, g_wcat)

        self._fork(dev, "fork3", props, head_reduce)
        join(dev, side)
        return res
