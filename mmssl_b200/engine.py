"""Forward / backward schedule of the MMSSL hot path on the CUDA library.

Implements the closed form of ``MMSSL.forward`` (reference Models.py:171-220; SURVEY.md appendix A)
and its hand-derived backward as an explicit sequence of library kernels.  No autograd inside:
``functional.MMSSLForwardFn`` wraps it for the drop-in ``Models.MMSSL`` and ``hotstep.HotStep``
drives it directly (fused with the loss kernels and AdamW, CUDA-graph captured).

Launch inventory of one forward (K GCN layers, modality graphs aliasing ui/iu as at step 0,
main.py:68-69):  2 projections x (split, GEMM, epilogue) + 2 two-RHS SpMM (image|text batched)
+ 2 id SpMM + Wsum + 2 fused id-fusion kernels + 2K SpMM (softmax / layer-sum fused) + 2 combine kernels,
scheduled on three streams (see ``Engine.two_streams``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import os

import torch

from . import ops
from .graph import BipartiteGraph

P_WV, P_BV, P_WT, P_BT = "image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias"
P_EU, P_EI, P_WCAT = "user_id_embedding.weight", "item_id_embedding.weight", "weight_dict.w_self_attention_cat"
LIVE = (P_WV, P_BV, P_WT, P_BT, P_EU, P_EI, P_WCAT)


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



def _prio(name: str, default: int) -> int:
    """Stream priority of one branch of the step (0 = lowest .. -5); MMSSL_PRIO_<NAME> overrides the measured default."""
    return int(os.environ.get("MMSSL_PRIO_" + name, default))


class Engine:
    def __init__(self, embed_size: int, n_layers: int, head_num: int = 4, id_cat_rate: float = 0.36,
                 model_cat_rate: float = 0.55, proj_impl: str = "tc"):
        if embed_size not in (64, 128, 256):
            raise ValueError("mmssl_b200 kernels are built for embed_size 64, 128 or 256")
        self.d, self.K, self.H = embed_size, n_layers, head_num
        self.id_rate, self.cat_rate = id_cat_rate, model_cat_rate
        self.proj_impl = proj_impl
        self._tile_id: Dict[Tuple, torch.Tensor] = {}
        # The modality branch (projection -> A_ui [Xv|Xt] -> A_iu [Uv|Ut]) and the id/GCN branch are
        # independent until the final combine (and again after combine-backward), so they run on two
        # streams; inside a CUDA graph they become parallel branches.  Set to False to serialise.
        self.two_streams = True
        self._side: Dict[Tuple, torch.cuda.Stream] = {}
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

    def _pair(self, dev, fn_a, fn_b):
        """Run two independent kernel groups concurrently (user side on the current stream, item side
        on the 'pair' stream) and join.  Returns (fn_a(), fn_b())."""
        if not self.two_streams:
            return fn_a(), fn_b()
        key = (dev.type, dev.index, "pair")
        st = self._side.get(key)
        if st is None:
            st = torch.cuda.Stream(device=dev, priority=_prio("PAIR", -1))      # twin of the critical id / GCN chain: ahead of the projection branch
            self._side[key] = st
        main = torch.cuda.current_stream(dev)
        st.wait_stream(main)
        with torch.cuda.stream(st):
            rb = fn_b()
        ra = fn_a()
        main.wait_stream(st)
        return ra, rb

    def _fork2(self, dev, fn_a, fn_b, name: str = "fork2"):
        """fn_a on the current stream, fn_b on a third stream (forked from / joined into the current one); serial when
        `two_streams` is off.  Used for the image | text halves of the projection, which are independent."""
        if not self.two_streams:
            fn_a(); fn_b()
            return
        key = (dev.type, dev.index, name)
        st = self._side.get(key)
        if st is None:
            st = torch.cuda.Stream(device=dev, priority=_prio("FORK", 0))
            self._side[key] = st
        cur = torch.cuda.current_stream(dev)
        st.wait_stream(cur)
        with torch.cuda.stream(st):
            fn_b()
        fn_a()
        cur.wait_stream(st)

    def _named_stream(self, dev, name: str) -> torch.cuda.Stream:
        """One more branch of the step (the caller forks it from and joins it into the main stream)."""
        key = (dev.type, dev.index, name)
        st = self._side.get(key)
        if st is None:
            st = torch.cuda.Stream(device=dev, priority=_prio(name.upper(), 0))
            self._side[key] = st
        return st

    def _side_stream(self, dev) -> torch.cuda.Stream:
        key = (dev.type, dev.index)
        st = self._side.get(key)
        if st is None:
            st = torch.cuda.Stream(device=dev, priority=_prio("SIDE", 0))
            self._side[key] = st
        return st

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
    def _project(self, w, b, fs: FeatureStore, mask, y, y_pre=None):
        I, d, D = fs.n_items, self.d, fs.dim
        if self.proj_impl == "tc":
            w_hi, w_lo = ops.split_bf16(w)
            floats, sk = ops.gemm_bf16x3_plan(I, d, D)
            part = self._new(floats, dev=y.device)
            ops.gemm_bf16x3(fs.hi, fs.lo, w_hi, w_lo, I, d, D, sk, part)
        else:
            if fs.fp32 is None:
                raise RuntimeError("proj_impl='simt' needs the fp32 features (keep_fp32=True)")
            sk = 1
            part = self._new(I, d, dev=y.device)
            ops.sgemm(fs.fp32, w, part, trans_b=True)
        ops.proj_epilogue(part, sk, I, d, b, mask, y, y_pre)

    def _project_bwd(self, gx, mask, fs: FeatureStore, dw, db):
        """dW[d,D] = (gx*mask)^T F ; db = colsum(gx*mask)."""
        I, d, D = fs.n_items, self.d, fs.dim
        if self.proj_impl == "tc":
            g_hi, g_lo = ops.split_bf16_t(gx, mask, ldo=fs.t_hi.shape[1], colsum=db)   # [d, ceil8(I)]; db from the same pass
            floats, sk = ops.gemm_bf16x3_plan(D, d, I)
            part = self._new(floats, dev=gx.device)
            ops.gemm_bf16x3(fs.t_hi, fs.t_lo, g_hi, g_lo, D, d, I, sk, part)
            ops.wgrad_epilogue(part, sk, D, d, dw)
        else:
            gm = self._new(I, d, dev=gx.device)
            ops.mul_mask(gx, mask, gm)
            ops.sgemm(gm, fs.fp32, dw, trans_a=True)
            ops.colsum(gx, mask, db)

    # ------------------------------------------------------------------ forward
    def forward(self, P: Dict[str, torch.Tensor], feats: Tuple[FeatureStore, FeatureStore],
                graphs: Sequence[BipartiteGraph], masks, want_sumsq: bool = True, side_pre=None):
        """masks: None, a pair of [I, d] keep-masks (0 or 1/(1-p)), or a callable returning one -- the
        callable and `side_pre` run at the head of the modality branch, i.e. off the critical path."""
        g_ui, g_iu, g_vui, g_viu, g_tui, g_tiu = graphs
        U, I = g_ui.shape
        d, K = self.d, self.K
        e_u, e_i = P[P_EU], P[P_EI]
        dev = e_u.device
        X2, U2, I2 = self._new(I, 2 * d, dev=dev), self._new(U, 2 * d, dev=dev), self._new(I, 2 * d, dev=dev)
        xv, xt = X2[:, :d], X2[:, d:]
        uv, ut = U2[:, :d], U2[:, d:]
        iv, it = I2[:, :d], I2[:, d:]
        main = torch.cuda.current_stream(dev)
        side = self._side_stream(dev) if self.two_streams else main

        resolved = [masks]

        def modal_branch():
            if side_pre is not None:
                side_pre()
            m = masks() if callable(masks) else masks
            resolved[0] = m
            # the two projections are independent HBM streams (118 + 30 MB at Baby): side by side on two streams
            self._fork2(dev, lambda: self._project(P[P_WV], P[P_BV], feats[0], m[0] if m else None, xv),    # Models.py:173
                        lambda: self._project(P[P_WT], P[P_BT], feats[1], m[1] if m else None, xt))         # Models.py:174
            self._spmm(g_ui, "fwd", [xv, xt], "i", [uv, ut])                        # :177,182
            self._spmm(g_iu, "fwd", [uv, ut], "u", [iv, it])                        # :178,183

        if side is not main:
            side.wait_stream(main)
            with torch.cuda.stream(side):
                modal_branch()
        else:
            modal_branch()

        def id_prop(ga, gb, e, rows, space):                                           # :179-180,185-186
            def one(g):
                if g.nnz == 0:
                    return torch.zeros(rows, d, dtype=torch.float32, device=dev)
                return self._spmm(g, "fwd", [e], space)[0]
            ya = one(ga)
            return (ya, ya) if ga is gb else (ya, one(gb))

        (uvid, utid), (ivid, itid) = self._pair(dev, lambda: id_prop(g_vui, g_tui, e_i, U, "i"), lambda: id_prop(g_viu, g_tiu, e_u, I, "u"))
        st = FwdState(tuple(graphs), resolved[0], X2, U2, I2, (uvid, utid, ivid, itid),
                      fused=any(g.nnz > 0 for g in (g_vui, g_viu, g_tui, g_tiu)))
        if st.fused:                                                                   # :188-197 (closed form)
            if d in (64, 128):      # fused row x matrix kernels, Wsum in shared memory
                st.wsum, st.wsum_t = ops.wsum(P[P_WCAT], d, self.H)

                def fuse(ya, yb, e):
                    return ops.id_fuse2_fwd(ya, None if ya is yb else yb, 1.0 if ya is yb else 0.5, st.wsum, e, self.id_rate)
            else:                   # d = 256: the d x d matrix does not fit shared memory -> GEMM path
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

            (u0, st.zn_u, st.nrm_u), (i0, st.zn_i, st.nrm_i) = self._pair(dev, lambda: fuse(uvid, utid, e_u), lambda: fuse(ivid, itid, e_i))
        else:
            u0, i0 = e_u, e_i
        # GCN layers: u_{k+1} = A_ui i_k ; i_{k+1} = A_iu u_{k+1}; softmax on the last one (:201-211);
        # the layer sums S_u, S_i accumulate in the SpMM epilogue (:213-214)
        s_u, s_i = self._new(U, d, dev=dev), self._new(I, d, dev=dev)
        cur_i = i0
        if K == 0:
            ops.axpby(u0, 1.0, 0.0, s_u)
            ops.axpby(i0, 1.0, 0.0, s_i)
        for k in range(K):
            last = k == K - 1
            epi = ops.EPI_SOFTMAX if last else ops.EPI_NONE
            mode = 2 if k == 0 else 1
            u_n = self._spmm(g_ui, "fwd", [cur_i], "i", epilogue=epi, ss=[s_u], s_mode=mode, sbases=[u0] if k == 0 else None)[0]
            i_n = self._spmm(g_iu, "fwd", [u_n], "u", epilogue=epi, ss=[s_i], s_mode=mode, sbases=[i0] if k == 0 else None)[0]
            if last:
                st.u_last, st.i_last = u_n, i_n
            cur_i = i_n
        inv = 1.0 / (K + 1)
        if side is not main:
            main.wait_stream(side)      # join: the combine needs Uv|Ut and Iv|It
        (u_f, st.sumsq_u), (i_f, st.sumsq_i) = self._pair(
            dev, lambda: ops.combine_fwd(s_u, uv, ut, inv, self.cat_rate, self._new(U, d, dev=dev), want_sumsq),      # :213,217
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
        self._pair(dev, lambda: ops.combine_bwd(g_uf, uv, ut, g_uv, g_ut, self.cat_rate, feat_reg_coef, gU2[:, :d], gU2[:, d:]),
                   lambda: ops.combine_bwd(g_if, iv, it, g_iv, g_it, self.cat_rate, feat_reg_coef, gI2[:, :d], gI2[:, d:]))
        main = torch.cuda.current_stream(dev)
        side = self._side_stream(dev) if self.two_streams else main
        w_slots = (slot(P_WV, P[P_WV]), slot(P_BV, P[P_BV]), slot(P_WT, P[P_WT]), slot(P_BT, P[P_BT]))

        def modal_backward():
            # modality propagation backward (Models.py:177-178,182-183), image|text batched, then the
            # projection backward (dropout mask folded into the operand split)
            self._spmm(g_iu, "bwd", [gI2[:, :d], gI2[:, d:]], "i", [gU2[:, :d], gU2[:, d:]], cs=[gU2[:, :d], gU2[:, d:]], alpha=1.0)
            gX2 = self._new(I, 2 * d, dev=dev)
            self._spmm(g_ui, "bwd", [gU2[:, :d], gU2[:, d:]], "u", [gX2[:, :d], gX2[:, d:]])
            m = st.masks
            self._fork2(dev, lambda: self._project_bwd(gX2[:, :d], m[0] if m else None, feats[0], w_slots[0], w_slots[1]),
                        lambda: self._project_bwd(gX2[:, d:], m[1] if m else None, feats[1], w_slots[2], w_slots[3]))
            return gX2

        if side is not main:
            side.wait_stream(main)
            with torch.cuda.stream(side):
                keep = modal_backward()
        else:
            keep = modal_backward()
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

            _, (gt_uvid, gt_utid, part_u) = self._pair(dev, chain, user_side)
            gt_ivid, gt_itid, part_i = fuse_bwd2(g_ei, st.zn_i, st.nrm_i, ivid, itid, g_ivid, g_itid)
            dwcat_args = (part_u, part_i)
        else:
            self._pair(dev, chain, lambda: ops.axpby(g_uf, inv, 0.0, g_eu))
        if fused2:
            pass
        elif st.fused:
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
                    tb = ta.clone() if g_yb is not None or g_ya is not None else ta
                    if g_ya is not None:
                        ops.axpby(g_ya, 1.0, 1.0, ta)
                    if g_yb is not None:
                        ops.axpby(g_yb, 1.0, 1.0, tb)
                return ta, tb

            gt_uvid, gt_utid = fuse_bwd(g_eu, st.zn_u, st.nrm_u, uvid, utid, g_uvid, g_utid, U)
            gt_ivid, gt_itid = fuse_bwd(g_ei, st.zn_i, st.nrm_i, ivid, itid, g_ivid, g_itid, I)
            ops.sgemm(self._tile(dev), d_wsum, g_wcat, trans_a=True)            # dWcat[h] = dWsum for every head
        else:
            g_wcat.zero_()
            gt_uvid, gt_utid, gt_ivid, gt_itid = g_uvid, g_utid, g_ivid, g_itid

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
            self._pair(dev, lambda: id_prop_bwd(g_vui, g_tui, gt_uvid, gt_utid, g_ei, st.fused and uvid is utid, "u"),
                       lambda: id_prop_bwd(g_viu, g_tiu, gt_ivid, gt_itid, g_eu, st.fused and ivid is itid, "i"))

        def head_reduce():
            if dwcat_args is not None:
                ops.dwcat_reduce(dwcat_args[0], dwcat_args[1], d, self.H, g_wcat)

        self._fork2(dev, props, head_reduce, name="fork3")
        if side is not main:
            main.wait_stream(side)
        return res
