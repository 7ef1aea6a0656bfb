"""The reference's whole training iteration on the device (SURVEY 8f "next" #2): the body of the batch loop of
``Trainer.train`` (main.py:333-434) -- Discriminator step, generator step with the ``G_rate * G_lossf`` term, both
optimisers, and the top-k bookkeeping that rebuilds the modality graphs -- as one sequence of library kernels.

What the reference does per iteration and what runs here instead:
  main.py:339-342  forward under no_grad                        -> Engine.forward (same kernels as the hot step)
  main.py:343-345  3x u_sim_calculation (dense [B, I] rows)     -> gan.u_sim_forward (GEMM + mask/normalise kernel)
  main.py:346-361  D(fake), Gumbel "real" rows built from a scipy .todense() copied to the GPU, D(real), gradient
                   penalty (autograd double backward), Adam     -> gan.d_step: closed-form sweeps, no autograd, the
                                                                   training rows read from the CSR on the device
  main.py:363-371  forward + BPR                                -> HotStep (fused loss kernels)
  main.py:372-375  2x u_sim_calculation with grad               -> gan.u_sim_forward / u_sim_backward
  main.py:378-405  scipy / python-list graph bookkeeping with 2 device->host copies per step
                                                                -> regraph kernels: top-k, pair lists and degree
                                                                   normalisation stay on the GPU, CSR built by
                                                                   mmssl_csr_from_coo
  main.py:408-420  feat_reg, 2x InfoNCE, D(G_inputf), loss      -> HotStep + gan.g_side (input gradient only)
  main.py:427-434  backward, AdamW, 4 float() host syncs        -> Engine.backward + mmssl_adamw; losses stay on the device

Reference quirks kept (oracle/gan_oracle.py:FullStep is the specification, pinned to a recorded trace of the unmodified
trainer): with the default ``T = 1`` the first iteration of an epoch collects pairs, the second builds the graphs from them,
every later one rebuilds from empty lists (nnz = 0 graphs); the pair lists tile the user vector against row-major ids;
the new graphs take effect from the NEXT iteration's first forward.

Randomness: the reference draws the dropout masks of the model and of D, the Gumbel uniforms and the penalty's
interpolation weights from torch's global generators.  ``step`` takes all of them as optional arguments (tests inject the
recorded draws); anything not given is drawn on the device from torch's CUDA generator.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import _lib, gan
from ._lib import ptr, stream
from .engine import LIVE, FeatureStore, capture_graph
from .graph import BipartiteGraph
from .hotstep import HotStep, HotStepConfig


@dataclass
class FullStepConfig:
    hot: HotStepConfig = field(default_factory=HotStepConfig)
    gan: gan.GanHyper = field(default_factory=gan.GanHyper)
    m_topk_rate: float = 1e-4       # parser.py:98
    T: int = 1                      # parser.py:93
    G_drop1: float = 0.31           # parser.py:84
    G_drop2: float = 0.5            # parser.py:85


# ------------------------------------------------------------------------------------------ regraph ops
def topk_rows(x: torch.Tensor, k: int) -> torch.Tensor:
    """ids[rows, k] of the k largest entries per row, best first (torch.topk at main.py:397,400)."""
    lib = _lib.load(require_device=True)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    ids = torch.empty(x.shape[0], k, dtype=torch.int64, device=x.device)
    _lib.check(lib.mmssl_topk_rows(ptr(x), x.stride(0), x.shape[0], x.shape[1], int(k), ptr(ids), stream()))
    return ids


def pair_append(users: torch.Tensor, ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(x, y) of main.py:398-402 for one modality and one step."""
    lib = _lib.load(require_device=True)
    B, k = ids.shape
    x = torch.empty(B * k, dtype=torch.int64, device=ids.device)
    y = torch.empty(B * k, dtype=torch.int64, device=ids.device)
    _lib.check(lib.mmssl_pair_append(ptr(users), B, ptr(ids), k, ptr(x), ptr(y), stream()))
    return x, y


def degree_values(idx: torch.Tensor, n_rows: int) -> torch.Tensor:
    lib = _lib.load(require_device=True)
    vals = torch.empty(idx.numel(), dtype=torch.float32, device=idx.device)
    scratch = torch.empty(max(n_rows, 1), dtype=torch.int32, device=idx.device)
    _lib.check(lib.mmssl_degree_values(ptr(idx), idx.numel(), n_rows, ptr(scratch), ptr(vals), stream()))
    return vals


def graphs_from_pairs(x: torch.Tensor, y: torch.Tensor, n_users: int, n_items: int) -> Tuple[BipartiteGraph, BipartiteGraph]:
    """main.py:379-391 for one modality: csr_norm(M), csr_norm(M^T) with M = the 0/1 pair matrix, duplicates summed."""
    ui = BipartiteGraph(x, y, degree_values(x, n_users), (n_users, n_items), tighten=False)
    iu = BipartiteGraph(y, x, degree_values(y, n_items), (n_items, n_users), tighten=False)
    return ui, iu


# ------------------------------------------------------------------------------------------ the step
class FullStep:
    """``FullStep(params, d_state, feats, train_indptr, train_indices, ui_graph, iu_graph, cfg, batch)`` then ``step(...)``
    once per batch.  ``params``: the live MMSSL parameters under their state_dict names (updated in place);
    ``d_state``: ``Discriminator(n_items).state_dict()`` (updated in place); ``train_indptr/indices``: the training
    interactions as int64 CSR with sorted rows (``ui_graph_raw``, main.py:58)."""

    def __init__(self, params: Dict[str, torch.Tensor], d_state: Dict[str, torch.Tensor], feats: Sequence[FeatureStore],
                 train_indptr: torch.Tensor, train_indices: torch.Tensor, ui_graph: BipartiteGraph, iu_graph: BipartiteGraph,
                 cfg: FullStepConfig, batch: int, ops_namespace=None):
        if ops_namespace is None:
            from . import gan_ops as ops_namespace       # raises without the extension / a CUDA device
        self.K = ops_namespace
        self.cfg = cfg
        self.U, self.I = ui_graph.shape
        self.batch = batch
        self.indptr, self.indices = train_indptr, train_indices
        graphs = [ui_graph, iu_graph, ui_graph, iu_graph, ui_graph, iu_graph]          # main.py:68-69
        self.hs = HotStep(params, feats, graphs, cfg.hot, batch=batch, optimizer_step=True, allow_alias=False)
        self.hs.post_forward = self._generator_side
        self.D = gan.DiscriminatorState(d_state)
        if hasattr(self.K, "register_weights"):          # tensor-core route: the weights' bf16 splits are cached per optimiser step
            self.K.register_weights([self.D.t["net.0.weight"], self.D.t["net.4.weight"]])
        self.idx = 0                                    # iteration inside the epoch (main.py:333)
        self.pairs: Dict[str, List[Tuple[torch.Tensor, torch.Tensor]]] = {"image": [], "text": []}
        # (x, y) pair lists the current modality graphs were built from; None: still the training graphs of step 0
        self.graph_pairs: Dict[str, Optional[Tuple[torch.Tensor, torch.Tensor]]] = {"image": None, "text": None}
        self.k = int(self.I * cfg.m_topk_rate)
        dev = self.hs.P[LIVE[0]].device
        f = dict(dtype=torch.float32, device=dev)
        d = cfg.hot.embed_size
        # gradient tables of the G_rate * G_lossf term w.r.t. Iv, It, Uv, Ut: one buffer, one memset per step
        self.gsim = torch.zeros(2 * (self.U + self.I) * d, **f)
        o = 0
        self.g_iv = self.gsim[o:o + self.I * d].view(self.I, d); o += self.I * d
        self.g_it = self.gsim[o:o + self.I * d].view(self.I, d); o += self.I * d
        self.g_uv = self.gsim[o:o + self.U * d].view(self.U, d); o += self.U * d
        self.g_ut = self.gsim[o:o + self.U * d].view(self.U, d)
        self.h1, self.h2 = d_state["net.0.weight"].shape[0], d_state["net.4.weight"].shape[0]
        self._draw: Dict[str, object] = {}
        self.last: Dict[str, torch.Tensor] = {}

    # -------------------------------------------------------------- epoch boundary (main.py:325-333)
    def start_epoch(self) -> None:
        self.idx = 0

    # -------------------------------------------------------------- random draws
    def _mask(self, shape, p: float) -> torch.Tensor:
        dev = self.gsim.device
        return F.dropout(torch.ones(*shape, dtype=torch.float32, device=dev), p, True)

    def _draws(self, model_masks, d_masks1, d_masks2, gumbel_u, alpha):
        B, I, d = self.batch, self.I, self.cfg.hot.embed_size
        dev = self.gsim.device
        p = self.cfg.hot.drop_rate
        if model_masks is None:          # order of consumption in the reference: forward 1 (image, text), forward 2
            model_masks = [self._mask((I, d), p) for _ in range(4)]
        if gumbel_u is None:
            gumbel_u = torch.rand(B, I, dtype=torch.float32, device=dev)
        if d_masks1 is None:
            d_masks1 = [self._mask((2 * B, self.h1), self.cfg.G_drop1) for _ in range(4)]
        if d_masks2 is None:
            d_masks2 = [self._mask((2 * B, self.h2), self.cfg.G_drop2) for _ in range(4)]
        if alpha is None:
            alpha = torch.rand(2 * B, dtype=torch.float32, device=dev)
        return model_masks, d_masks1, d_masks2, gumbel_u, alpha.reshape(-1)

    # -------------------------------------------------------------- generator side (called by HotStep between loss and backward)
    def _generator_side(self, outs, st):
        K, hp = self.K, self.cfg.gan
        _, _, iv, it, uv, ut = outs[:6]
        users = self.hs.idx[0]
        self.gsim.zero_()
        c_img = gan.u_sim_forward(K, uv, iv, users, self.indptr, self.indices)          # main.py:372
        c_txt = gan.u_sim_forward(K, ut, it, users, self.indptr, self.indices)          # main.py:373
        self._bookkeeping(users, c_img["y"], c_txt["y"])                                # main.py:378-405
        s_sum, dx_img, dx_txt = gan.g_side(K, self.D, hp, c_img, c_txt, self._draw["m1"][3], self._draw["m2"][3])   # :414-418
        gan.u_sim_backward(K, c_img, dx_img, iv, self.indptr, self.indices, self.g_uv, self.g_iv)
        gan.u_sim_backward(K, c_txt, dx_txt, it, self.indptr, self.indices, self.g_ut, self.g_it)
        self.last["G_s_sum"] = s_sum
        self.last["G_u_sim"] = (c_img["y"], c_txt["y"])
        return self.g_iv, self.g_it, self.g_uv, self.g_ut

    def _bookkeeping(self, users, img_sim, txt_sim) -> None:
        self._new_graphs = None
        if self.idx % self.cfg.T == 0 and self.idx != 0:
            if not self.pairs["image"] and not self.pairs["text"] and all(g.nnz == 0 for g in self.hs.graphs[2:]):
                return                                   # empty lists onto already empty graphs: nothing changes (steady state at T = 1)
            new = list(self.hs.graphs)
            self._new_pairs = {}
            for j, key in ((2, "image"), (4, "text")):
                xs = [p[0] for p in self.pairs[key]]
                ys = [p[1] for p in self.pairs[key]]
                e = torch.zeros(0, dtype=torch.int64, device=users.device)
                x = torch.cat(xs) if xs else e
                y = torch.cat(ys) if ys else e
                new[j], new[j + 1] = graphs_from_pairs(x, y, self.U, self.I)
                self._new_pairs[key] = (x, y)
            self.pairs = {"image": [], "text": []}
            self._new_graphs = tuple(new)
        elif self.k > 0:
            for key, sim in (("image", img_sim), ("text", txt_sim)):
                self.pairs[key].append(pair_append(users, topk_rows(sim, self.k)))

    # -------------------------------------------------------------- one iteration
    def _body(self, mm, m1, m2, gu, al) -> Dict[str, torch.Tensor]:
        K, hp, hs = self.K, self.cfg.gan, self.hs
        u_dev = hs.idx[0]
        self._draw = {"m1": m1, "m2": m2}
        # ---- D step (main.py:339-361)
        outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, (mm[0], mm[1]), want_sumsq=False)
        ui = gan.u_sim_forward(K, outs[0], outs[1], u_dev, self.indptr, self.indices)["y"]
        img = gan.u_sim_forward(K, outs[4], outs[2], u_dev, self.indptr, self.indices)["y"]
        txt = gan.u_sim_forward(K, outs[5], outs[3], u_dev, self.indptr, self.indices)["y"]
        dres = gan.d_step(K, self.D, hp, img, txt, ui, u_dev, self.indptr, self.indices, gu, al, m1[:3], m2[:3])
        self.last["D_u_sim"] = (ui, img, txt)
        # ---- G step (main.py:363-429): HotStep.run calls _generator_side between the loss kernels and the backward
        hs.masks = (mm[2], mm[3])
        loss5 = hs.run()
        n = 2 * self.batch
        g_lossf = self.last["G_s_sum"] * (-100.0 / n)
        loss_d = (dres["lossf_sum"] - dres["lossr_sum"]) * (100.0 / n) + hp.gp_rate * dres["gp"]
        return dict(loss5=loss5, G_lossf=g_lossf, batch_loss=loss5[0] + hp.G_rate * g_lossf, gp=dres["gp"], loss_D=loss_d,
                    D_grads=dres["grads"])

    def step(self, users, pos, neg, model_masks: Optional[Sequence[torch.Tensor]] = None,
             d_masks1: Optional[Sequence[torch.Tensor]] = None, d_masks2: Optional[Sequence[torch.Tensor]] = None,
             gumbel_u: Optional[torch.Tensor] = None, alpha: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """users/pos/neg: the batch of ``data_generator.sample()`` (lists or int64 tensors).  Returns device tensors:
        ``loss5`` = [hot total, mf, emb, feat_reg, cl] (HotStep), ``G_lossf``, ``batch_loss`` (main.py:420), ``gp``,
        ``loss_D`` (main.py:357) -- nothing is copied to the host."""
        self.hs.set_indices(users, pos, neg)
        draws = self._draws(model_masks, d_masks1, d_masks2, gumbel_u, alpha)
        if self._graph is not None and self.steady():
            for dst, src in zip(self._flat(self._static), self._flat(draws)):
                dst.copy_(src)
            self._graph.replay()
            self.D.step += 1
            self.idx += 1
            return self._static_out
        out = self._body(*draws)
        if self._new_graphs is not None:
            self.hs.graphs = self._new_graphs
            self.graph_pairs = self._new_pairs
        self.idx += 1
        return out

    # -------------------------------------------------------------- checkpoint (checkpoint.py)
    def state_dict(self) -> dict:
        """HotStep state + the Discriminator and its Adam state + the epoch bookkeeping: iteration in the epoch, collected
        pairs, and the pair lists the modality graphs were built from (the graphs are rebuilt from them on load)."""
        st = self.hs.state_dict()
        st.update(kind="fullstep", D=self.D.state_dict(), D_optim=self.D.optim_state_dict(),
                  fullstep=dict(idx=int(self.idx), pairs={k: [tuple(p) for p in v] for k, v in self.pairs.items()},
                                graph_pairs=dict(self.graph_pairs)))
        return st

    def load_state_dict(self, state: dict) -> None:
        """In place, like HotStep.load_state_dict.  A captured iteration survives the load when the modality graphs stay the
        ones it was recorded with; otherwise it is dropped (Trainer re-captures once ``steady()`` holds again)."""
        from . import checkpoint
        checkpoint.check_format(state, ("fullstep", "trainer"))
        checkpoint.check_meta(state["meta"], self.hs.meta())
        fs = state["fullstep"]
        self.hs.load_state_dict(state)
        self.D.load_state_dict(state["D"], state["D_optim"])
        dev = self.gsim.device
        on = lambda p: (p[0].to(dev), p[1].to(dev))
        self.idx = int(fs["idx"])
        self.pairs = {k: [on(p) for p in fs["pairs"][k]] for k in ("image", "text")}
        want = {k: (None if fs["graph_pairs"][k] is None else on(fs["graph_pairs"][k])) for k in ("image", "text")}
        same = lambda a, b: (a is None and b is None) or (a is not None and b is not None and all(
            x.shape == y.shape and bool(torch.equal(x, y)) for x, y in zip(a, b)))
        if not all(same(want[k], self.graph_pairs[k]) for k in ("image", "text")):
            g = list(self.hs.graphs)
            for j, key in ((2, "image"), (4, "text")):
                if want[key] is None:                    # the training graphs, as at step 0 (main.py:68-69)
                    g[j], g[j + 1] = g[0], g[1]
                else:
                    g[j], g[j + 1] = graphs_from_pairs(want[key][0], want[key][1], self.U, self.I)
            self.hs.graphs = tuple(g)
            self.graph_pairs = want
            self._graph = None
        if hasattr(self.K, "refresh_weight_splits"):     # the bf16 splits of D's weights are cached (DESIGN section 9)
            self.K.refresh_weight_splits()

    # -------------------------------------------------------------- CUDA graph of the steady state
    _graph = None

    @staticmethod
    def _flat(draws):
        mm, m1, m2, gu, al = draws
        return [*mm, *m1, *m2, gu, al]

    def steady(self) -> bool:
        """True when an iteration leaves the graphs as they are and collects nothing: the modality graphs are empty, the pair
        lists are empty and this iteration is on the rebuild branch (with the default T = 1: every iteration from the 4th of
        an epoch on; with m_topk_rate * n_items < 1, as at Baby, from the 3rd of the FIRST epoch on, for the whole run)."""
        rebuild = self.idx % self.cfg.T == 0 and self.idx != 0
        empty = not self.pairs["image"] and not self.pairs["text"] and all(g.nnz == 0 for g in self.hs.graphs[2:])
        return empty and (rebuild or self.k == 0)

    def capture(self, keep_state: bool = False) -> None:
        """Capture one steady-state iteration (D step + G step + both optimisers, ~150 launches) into a CUDA graph; ``step``
        replays it whenever ``steady()`` holds and runs eagerly otherwise (first iterations of an epoch).  The random draws
        are static input buffers refilled before every replay (by torch's generator, or by the caller's injected draws).
        Green on the H100 (tests/test_gpu_zzz_gemm_wide.py::test_full_step_cuda_graph_replay_equals_eager).
        NOTE: the warm-up below is ONE REAL iteration on the indices currently in ``hs.idx`` with draws from torch's generator
        (both optimisers step, BatchNorm statistics move): call it where an iteration of the run belongs (trainer.py does), not
        in front of one.  ``keep_state=True`` undoes it instead: the parameters, both optimisers, BatchNorm statistics, counters
        and torch's generators are put back as they were before the capture (a resumed run whose saved run had already captured
        re-captures this way, so it does not train one iteration more than the uninterrupted run)."""
        from . import checkpoint
        if not self.steady():
            raise RuntimeError("capture() needs the steady state: run the first iterations of the epoch eagerly")
        dev = self.gsim.device
        if keep_state:
            snap, rng = checkpoint.clone_state(self.state_dict()), checkpoint.rng_state(dev)
        self._static = self._draws(None, None, None, None, None)

        def warm():
            self._body(*self._static)
            self.idx += 1

        def body():
            step_before = self.D.step
            out = self._body(*self._static)
            self.D.step = step_before                        # the capture pass does not execute
            return out

        self._graph, self._static_out = capture_graph(warm, body)
        if keep_state:                  # in place: the captured graph reads the same buffers (the modality graphs did not change)
            self.load_state_dict(snap)
            checkpoint.set_rng_state(rng, dev)
