"""Fused hot training step: forward -> BPR + 2x InfoNCE + feat_reg (value and gradient seeds in the
same kernels) -> hand-written backward -> multi-tensor AdamW, with static buffers, so the whole step
is captured once into a CUDA graph and replayed (no Python / launch overhead in the steady state, no
host synchronisation besides reading the loss).  Inside the graph the work forms three parallel
branches (engine.py): id/GCN chain, modality branch (projection + image|text propagation), and the
item-side twin of every user-side kernel; memset, dropout masks, the optional GPU sampler and BPR ride
on the side branches, off the critical path.

Reference unit of work (SURVEY.md 8d): main.py:363-371 (forward + BPR), :408-414 (feat_reg, InfoNCE),
:420 (loss without the GAN term), :427-429 (zero_grad / backward / AdamW step).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F

from . import checkpoint, ops
from .engine import LIVE, P_EI, P_EU, Engine, FeatureStore, capture_graph, join
from .graph import BipartiteGraph


@dataclass
class HotStepConfig:
    embed_size: int = 64
    n_layers: int = 2
    head_num: int = 4
    id_cat_rate: float = 0.36
    model_cat_rate: float = 0.55
    drop_rate: float = 0.2
    tau: float = 0.5
    cl_rate: float = 0.03
    emb_decay: float = 1e-5
    feat_reg_decay: float = 1e-5
    batch_size: int = 1024          # the *configured* batch size the BPR regulariser divides by (main.py:504)
    lr: float = 5.5e-4
    weight_decay: float = 1e-2
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    proj_impl: str = "tc"


class HotStep:
    def __init__(self, params: Dict[str, torch.Tensor], feats: Sequence[FeatureStore], graphs: Sequence[BipartiteGraph],
                 cfg: HotStepConfig, batch: int, optimizer_step: bool = True, sampler=None, allow_alias: bool = True):
        self.cfg = cfg
        self.P = {k: params[k] for k in LIVE}
        for k, t in self.P.items():
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), k
        self.feats, self.graphs = tuple(feats), tuple(graphs)
        self.engine = Engine(cfg.embed_size, cfg.n_layers, cfg.head_num, cfg.id_cat_rate, cfg.model_cat_rate, cfg.proj_impl)
        self.U, self.I = graphs[0].shape
        self.batch = batch
        self.optimizer_step = optimizer_step
        self.sampler = sampler          # optional sampler.DeviceTripleSampler: batches are drawn on the device
        if sampler is not None:
            sampler.reserve(batch)      # workspace of the multi-CTA path (batch > 1024) before any capture
        self.grad_sync = None           # optional callable run between backward and AdamW (data-parallel all-reduce)
        # optional callable(outs, st) -> (g_Iv, g_It, g_Uv, g_Ut): extra output gradients of the forward, e.g. the
        # G_rate * G_lossf term of the full step (main.py:414-420); runs after the loss kernels, before the backward
        self.post_forward = None
        dev = self.P[P_EU].device
        d = cfg.embed_size
        f = dict(dtype=torch.float32, device=dev)
        self.idx = torch.zeros(3, batch, dtype=torch.int64, device=dev)     # users / pos / neg (static input)
        # image and text graphs are the same object at step 0 (main.py:68-69): one InfoNCE instead of two.  The full
        # step (fullstep.py) replaces them by distinct top-k graphs later, so it asks for the general layout up front.
        self.alias_id = allow_alias and graphs[2] is graphs[4]
        # gradient seeds of the loss kernels: one contiguous buffer -> one memset per step
        n_u = 2 if self.alias_id else 3
        self.gflat = torch.zeros((n_u * self.U + self.I) * d, **f)
        self.g_uf = self.gflat[:self.U * d].view(self.U, d)
        self.g_uvid = self.gflat[self.U * d:2 * self.U * d].view(self.U, d)
        self.g_utid = self.g_uvid if self.alias_id else self.gflat[2 * self.U * d:3 * self.U * d].view(self.U, d)
        self.g_if = self.gflat[n_u * self.U * d:].view(self.I, d)
        self.ones = torch.ones(self.I, d, **f)
        self.nce = [ops.InfoNCEWork(batch, d, dev) for _ in range(1 if self.alias_id else 2)]
        self.cl_seed = torch.full((1,), cfg.cl_rate * (2.0 if self.alias_id else 1.0), **f)
        self.out5 = torch.zeros(5, **f)
        self.grads = {k: torch.zeros_like(t) for k, t in self.P.items()}
        self.m = {k: torch.zeros_like(t) for k, t in self.P.items()}
        self.v = {k: torch.zeros_like(t) for k, t in self.P.items()}
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.masks: Optional[tuple] = None          # injected dropout masks (tests); None -> torch RNG
        self.training = True
        self._graph: Optional[torch.cuda.CUDAGraph] = None

    # ------------------------------------------------------------------ one step on the current stream
    def _masks(self):
        if not self.training or self.cfg.drop_rate <= 0:
            return None
        if self.masks is not None:
            return self.masks
        p = self.cfg.drop_rate
        return (F.dropout(self.ones, p, True), F.dropout(self.ones, p, True))     # image first, like Models.py:173-174

    def run(self) -> torch.Tensor:
        """Executes one hot step with the indices currently in ``self.idx``; returns the device
        tensor [total, mf, emb, feat_reg, cl]."""
        cfg = self.cfg
        users, pos, neg = self.idx[0], self.idx[1], self.idx[2]
        # the seed-buffer memset and the dropout masks are only needed by the modality branch / the
        # loss kernels, so they run at the head of the side stream, off the critical path
        def side_pre():
            self.gflat.zero_()
            if self.sampler is not None:      # (seed, optimiser step) -> a fresh batch on every graph replay
                self.sampler.sample_into(self.idx, step_dev=self.step_dev)

        outs, st = self.engine.forward(self.P, self.feats, self.graphs, self._masks, want_sumsq=True, side_pre=side_pre)
        u_f, i_f, _, _, _, _, u_vid, u_tid, _, _ = outs
        reg_coef = cfg.emb_decay / cfg.batch_size
        # BPR: value partials + gradient rows scattered straight into the dense table gradients
        dev = u_f.device
        with self.engine.branch(dev, "side") as side:     # BPR runs next to InfoNCE (both only add into the seed buffers, atomically)
            bpr_part, n_bpr = ops.bpr(u_f, i_f, i_f, users, pos, neg, mode=3, reg_coef=reg_coef,
                                      g_u=self.g_uf, g_p=self.g_if, g_n=self.g_if)
        # InfoNCE(Uvid[users], u_f[users]) + InfoNCE(Utid[users], u_f[users])   (main.py:411-412)
        inv_tau = 1.0 / cfg.tau
        parts = []
        for w, z1, gz1 in zip(self.nce, (u_vid, u_tid), (self.g_uvid, self.g_utid)):
            parts.append(ops.infonce_forward(z1, u_f, users, inv_tau, w, g_loss=self.cl_seed))
            if st.fused:    # with empty modality graphs z1 == 0: the loss is a constant, all gradients vanish
                ops.infonce_backward(users, inv_tau, w, gz1, self.g_uf)
        join(dev, side)
        nce1 = parts[0]
        nce2 = parts[0] if self.alias_id else parts[1]
        # the five loss VALUES feed nothing of the backward: assembled on a stream of their own, joined at the end of the step
        with self.engine.branch(dev, "loss") as loss_st:
            ops.loss_assemble(bpr_part, n_bpr, self.batch, reg_coef, st.sumsq_u, st.sumsq_i, 0.5 * cfg.feat_reg_decay / self.I,
                              nce1, nce2, self.batch, cfg.cl_rate, self.out5)
        extra = self.post_forward(outs, st) if self.post_forward is not None else (None, None, None, None)
        grads = [self.g_uf, self.g_if, extra[0], extra[1], extra[2], extra[3],
                 self.g_uvid if st.fused else None, (None if self.alias_id else self.g_utid) if st.fused else None, None, None]
        self.engine.backward(st, self.P, self.feats, grads, feat_reg_coef=cfg.feat_reg_decay / self.I, out=self.grads)
        if self.grad_sync is not None:
            self.grad_sync()
        if self.optimizer_step:
            ops.step_tick(self.step_dev)
            keys = list(LIVE)
            ops.adamw([self.P[k] for k in keys], [self.grads[k] for k in keys], [self.m[k] for k in keys],
                      [self.v[k] for k in keys], self.step_dev, cfg.lr, cfg.beta1, cfg.beta2, cfg.eps, cfg.weight_decay)
        join(dev, loss_st)
        return self.out5

    # ------------------------------------------------------------------ CUDA graph
    def capture(self, warmup: int = 2) -> None:
        """Capture ``run`` into a CUDA graph (static buffers; update ``self.idx`` between replays).
        Warm-up steps run on a side stream first and DO advance the optimiser state."""
        def warm():
            for _ in range(warmup):
                self.run()
        self._graph, _ = capture_graph(warm, self.run)

    def replay(self) -> torch.Tensor:
        if self._graph is None:
            raise RuntimeError("call capture() first")
        self._graph.replay()
        return self.out5

    # ------------------------------------------------------------------ checkpoint (checkpoint.py)
    _fingerprint = None

    def meta(self) -> dict:
        if self._fingerprint is None:        # the training graph (graphs[0]) never changes: one device->host copy per step object
            self._fingerprint = checkpoint.graph_fingerprint(self.graphs[0])
        m = checkpoint.make_meta(self.U, self.I, self.cfg, self.batch, self.feats, self._fingerprint)
        if self.sampler is not None:         # with (seed, step_dev) the device sampler's batches are fixed
            m["sampler_seed"] = int(self.sampler.seed)
        return m

    def state_dict(self) -> dict:
        """Parameters (reference keys), AdamW moments and step counter.  Tensors are the live buffers, not copies."""
        return dict(format=checkpoint.FORMAT, kind="hotstep", meta=self.meta(), model=dict(self.P),
                    optim=dict(m=dict(self.m), v=dict(self.v), step=int(self.step_dev.cpu()[0])))

    def load_state_dict(self, state: dict) -> None:
        """Copies a checkpoint (this step's, a FullStep's / Trainer's, or a row-sharded one read at world 1) into the live
        buffers in place: a graph captured before the load replays from the loaded state."""
        checkpoint.check_format(state, ("hotstep", "fullstep", "trainer"))
        checkpoint.check_meta(state["meta"], self.meta())
        model = {k: state["model"][k] for k in LIVE if k in state["model"]}
        checkpoint.copy_into(self.P, model, "model")
        checkpoint.copy_into(self.m, state["optim"]["m"], "optim.m")
        checkpoint.copy_into(self.v, state["optim"]["v"], "optim.v")
        self.step_dev.fill_(int(state["optim"]["step"]))

    def set_indices(self, users, pos, neg) -> None:
        """Device-side copy of one batch of triples into the static index buffer."""
        self.idx[0].copy_(torch.as_tensor(users, dtype=torch.int64), non_blocking=True)
        self.idx[1].copy_(torch.as_tensor(pos, dtype=torch.int64), non_blocking=True)
        self.idx[2].copy_(torch.as_tensor(neg, dtype=torch.int64), non_blocking=True)
