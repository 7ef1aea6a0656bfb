"""Mirror of the reference's ``Trainer`` (MMSSL/main.py:31-306, :308-498) over the device-resident full step.

Same life cycle as ``python main.py --dataset X``: ``Trainer(data, args)`` builds the model and the discriminator with the
reference's parameter-creation order (``set_seed`` then MMSSL then Discriminator + ``weights_init``: identical initial values
for the same seed), ``train()`` runs the epoch loop with the reference's batch count, evaluation cadence, best-recall /
early-stopping rule and log lines, ``test(users, is_val)`` is ``Trainer.test``.  What differs is what executes:

  main.py:333-434   the batch loop body         -> fullstep.FullStep.step   (one sequence of library kernels, no autograd,
                                                   no scipy / .cpu() / float() per step; losses accumulate on the device)
  main.py:301-306   Trainer.test -> test_torch  -> Engine.forward (eval) + evaluate.Evaluator (fused rank + metrics kernel)
  load_data.py:153  Data.sample                 -> ``sampler="reference"``: the same draws from `random` / `numpy.random`
                                                   (bit-identical batches for the same seeds, pinned to the reference in
                                                   tests/golden/sampler_small.json); ``sampler="device"``: the GPU sampler
                                                   kernel (no host work per step)
  load_data.py:10-88, main.py:54-58             -> dataset.ReferenceDataset (same files, same dictionaries)

``TrainerArgs`` carries the reference's flags with its defaults (utility/parser.py); an ``argparse.Namespace`` from the
reference's own ``parse_args()`` works as well (same attribute names)."""
from __future__ import annotations

import math
import random as rd
from dataclasses import dataclass
from time import time
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import checkpoint, gan
from .dataset import ReferenceDataset
from .engine import LIVE
from .evaluate import Evaluator
from .fullstep import FullStep, FullStepConfig
from .graph import BipartiteGraph
from .hotstep import HotStepConfig
from .synthetic import csr_norm


@dataclass
class TrainerArgs:
    """utility/parser.py defaults of every flag the training / evaluation loop reads (line numbers of the reference)."""
    dataset: str = ""
    seed: int = 2022                    # :51
    epoch: int = 1000                   # :53
    batch_size: int = 1024              # :54
    embed_size: int = 64                # :55
    D_lr: float = 3e-4                  # :56
    cl_rate: float = 0.03               # :60
    Ks: str = "[10, 20, 50]"            # :63
    regs: str = "[1e-5,1e-5,1e-2]"      # :64
    lr: float = 0.00055                 # :65
    drop_rate: float = 0.2              # :72
    model_cat_rate: float = 0.55        # :73
    id_cat_rate: float = 0.36           # :75
    head_num: int = 4                   # :77
    weight_size: str = "[64, 64]"       # :82
    G_rate: float = 1e-4                # :83
    G_drop1: float = 0.31               # :84
    G_drop2: float = 0.5                # :85
    gp_rate: float = 1.0                # :86
    real_data_tau: float = 0.005        # :88
    ui_pre_scale: float = 100.0         # :89
    T: int = 1                          # :93
    tau: float = 0.5                    # :94
    m_topk_rate: float = 1e-4           # :98
    log_log_scale: float = 1e-5         # :99
    verbose: int = 5                    # :8
    early_stopping_patience: int = 7    # :11
    feat_reg_decay: float = 1e-5        # :29
    mess_dropout: str = "[0.1, 0.1]"    # :13
    test_flag: str = "part"             # :16
    checkpoint: str = ""                # not in the reference: train() writes Trainer.save(checkpoint) after every epoch when set


def set_seed(seed: int) -> None:
    """main.py:520-524"""
    np.random.seed(seed)
    rd.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def reference_sample(data: ReferenceDataset, batch_size: int, n_items: Optional[int] = None) -> Tuple[List[int], List[int], List[int]]:
    """``Data.sample`` (utility/load_data.py:153-191): the same calls on the same global generators in the same order,
    so a run seeded like the reference draws the reference's batches.  ``n_items`` bounds the negatives (default: the
    loader's count, like the reference; the trainer passes the width of ``train_mat`` -- where the json files name an item
    id beyond it the reference would index its embedding table out of range)."""
    n_items = data.n_items if n_items is None else n_items
    if batch_size <= data.n_users:
        users = rd.sample(data.exist_users, batch_size)
    else:
        users = [rd.choice(data.exist_users) for _ in range(batch_size)]
    pos_items, neg_items = [], []
    for u in users:
        row = data.train_items[u]
        pos_items.append(row[np.random.randint(low=0, high=len(row), size=1)[0]])       # one positive: never a repeat
        while True:
            neg = np.random.randint(low=0, high=n_items, size=1)[0]
            if neg not in row:
                neg_items.append(int(neg))
                break
    return users, [int(p) for p in pos_items], neg_items


class Trainer:
    def __init__(self, data: ReferenceDataset, args=None, device: str = "cuda", sampler: str = "reference",
                 log: Optional[Callable[[str], None]] = print, proj_impl: str = "tc", cuda_graph: bool = False):
        import mmssl_b200.Models as M
        self.args = args = args if args is not None else TrainerArgs()
        self.data, self.log, self.device = data, (log or (lambda s: None)), torch.device(device)
        for k in ("embed_size", "head_num", "id_cat_rate", "model_cat_rate", "drop_rate", "G_drop1", "G_drop2"):
            setattr(M.args, k, getattr(args, k))                  # Models.py reads the module-global args (Models.py:13-15)
        self.batch_size = args.batch_size
        self.weight_size = eval(args.weight_size)
        self.n_layers = len(self.weight_size)
        self.decay = eval(args.regs)[0]                           # main.py:51-52
        self.Ks = eval(args.Ks)
        R = data.train_mat.tocsr().astype(np.float32)
        R.sum_duplicates()             # the device GAN path reads rows as sorted, duplicate-free index lists ...
        R.sort_indices()
        if R.nnz and not bool((R.data == 1).all()):
            raise ValueError("train_mat must be a 0/1 interaction matrix (the reference's todense() path would use its values; "
                             "the device path of the GAN side reads the sparsity pattern)")
        self.ui_graph_raw = R
        self.n_users, self.n_items = R.shape                      # main.py:63-64 (from train_mat, not from the json files)
        # main.py:70-74: model, .cuda(), discriminator, kaiming init of its Linear layers
        self.model = M.MMSSL(self.n_users, self.n_items, args.embed_size, self.weight_size, eval(args.mess_dropout),
                             np.asarray(data.image_feats), np.asarray(data.text_feats), proj_impl=proj_impl).to(self.device)
        self.D = M.Discriminator(self.n_items).to(self.device)
        self.D.apply(self._weights_init)
        dev = self.device
        t64 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int64)).to(dev)
        self.ui_graph = BipartiteGraph.from_scipy(csr_norm(R), device=dev)                       # main.py:66
        self.iu_graph = BipartiteGraph.from_scipy(csr_norm(R.T.tocsr()), device=dev)             # main.py:67
        named = dict(self.model.named_parameters())
        self.P = {k: named[k].data for k in LIVE}                 # updated in place: the nn.Module stays the checkpoint
        self.d_state = {k: v.data if isinstance(v, nn.Parameter) else v for k, v in self.D.state_dict(keep_vars=True).items()}
        hot = HotStepConfig(embed_size=args.embed_size, n_layers=self.n_layers, head_num=args.head_num, id_cat_rate=args.id_cat_rate,
                            model_cat_rate=args.model_cat_rate, drop_rate=args.drop_rate, tau=args.tau, cl_rate=args.cl_rate,
                            emb_decay=self.decay, feat_reg_decay=args.feat_reg_decay, batch_size=args.batch_size, lr=args.lr,
                            proj_impl=proj_impl)
        hp = gan.GanHyper(gp_rate=args.gp_rate, G_rate=args.G_rate, D_lr=args.D_lr, log_log_scale=args.log_log_scale,
                          real_data_tau=args.real_data_tau, ui_pre_scale=args.ui_pre_scale)
        cfg = FullStepConfig(hot=hot, gan=hp, m_topk_rate=args.m_topk_rate, T=args.T, G_drop1=args.G_drop1, G_drop2=args.G_drop2)
        self.step = FullStep(self.P, self.d_state, self.model._feature_stores(), t64(R.indptr), t64(R.indices), self.ui_graph,
                             self.iu_graph, cfg, batch=args.batch_size)
        self.evaluator = Evaluator(data.train_items, data.test_set, data.val_set, self.n_users, self.n_items, self.Ks, device=dev,
                                   test_flag=args.test_flag)
        if sampler == "device":
            from .sampler import DeviceTripleSampler
            self._dev_sampler = DeviceTripleSampler(R, device=dev, seed=args.seed)
            self._triples = torch.empty(3, args.batch_size, dtype=torch.int64, device=dev)
        elif sampler != "reference":
            raise ValueError("sampler must be 'reference' or 'device'")
        self.sampler = sampler
        self._n_sampled = 0
        # replay the steady-state iteration as one CUDA graph once the modality graphs have stopped changing
        # (FullStep.capture; experimental until its first GPU run -- off by default)
        self.cuda_graph = cuda_graph

    @staticmethod
    def _weights_init(m):                                          # main.py:133-136
        if isinstance(m, nn.Linear):
            nn.init.kaiming_normal_(m.weight)
            m.bias.data.fill_(0)

    # ------------------------------------------------------------------ main.py:301-306
    def test(self, users_to_test, is_val: bool) -> Dict[str, object]:
        hs = self.step.hs
        outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, None, want_sumsq=False)       # model.eval(): no dropout
        return self.evaluator.test_torch(outs[0], outs[1], users_to_test, is_val)

    def sample(self):
        if self.sampler == "device":
            self._dev_sampler.sample_into(self._triples, step=self._n_sampled)
            self._n_sampled += 1
            return self._triples[0], self._triples[1], self._triples[2]
        return reference_sample(self.data, self.batch_size, n_items=self.n_items)

    # ------------------------------------------------------------------ checkpoint (checkpoint.py)
    _loop: Optional[Dict[str, object]] = None        # epoch-loop state after the last finished epoch (what save() writes)
    _resume: Optional[Dict[str, object]] = None      # set by load(): where the next train() starts
    _capture_keeps_state = False                     # set by load(): see FullStep.capture(keep_state)

    def save(self, path: str) -> None:
        """Writes the whole training state at an epoch boundary: the model and the Discriminator under the reference's
        state_dict keys, both optimisers, the full step's epoch bookkeeping, the epoch loop's state, the sampler position and
        the RNG states.  ``load`` + ``train()`` continue the run at the next epoch."""
        st = self.step.state_dict()
        loop = dict(self._loop or dict(epoch=0, best_recall=0.0, stopping_step=0, test_ret=None, history=[], stopped=False))
        if loop["test_ret"] is not None:       # the evaluator's numpy arrays travel as tensors (the file loads with weights_only)
            loop["test_ret"] = {k: torch.from_numpy(v) if isinstance(v, np.ndarray) else v for k, v in loop["test_ret"].items()}
        st.update(kind="trainer", model=self.model.state_dict(), D=self.D.state_dict(),
                  trainer=dict(loop=loop, sampler=self.sampler, n_sampled=int(self._n_sampled), rng=checkpoint.rng_state(self.device),
                               sampler_seed=int(self._dev_sampler.seed) if self.sampler == "device" else None,
                               captured=self.step._graph is not None))
        checkpoint.save(st, path)

    def load(self, path: str) -> None:
        """Restores ``save(path)`` into this Trainer (built with the same data and shape arguments) in place."""
        st = checkpoint.load(path, kinds=("trainer",))
        checkpoint.check_meta(st["meta"], self.step.hs.meta())
        tr = st["trainer"]
        if tr["sampler"] != self.sampler:
            raise ValueError(f"checkpoint mismatch in sampler: saved {tr['sampler']!r}, this run {self.sampler!r}")
        if self.sampler == "device" and tr["sampler_seed"] != self._dev_sampler.seed:     # (seed, step) fixes the batches
            raise ValueError(f"checkpoint mismatch in sampler_seed: saved {tr['sampler_seed']}, this run {self._dev_sampler.seed}")
        self.model.load_state_dict(st["model"])          # in place: the unused registered parameters; the live ones and D below
        self.step.load_state_dict(st)
        self._n_sampled = int(tr["n_sampled"])
        loop = dict(tr["loop"])
        if loop["test_ret"] is not None:
            loop["test_ret"] = {k: v.numpy() if isinstance(v, torch.Tensor) else v for k, v in loop["test_ret"].items()}
        self._loop = self._resume = loop
        self.history = list(loop["history"])
        # the saved run had captured its steady-state iteration (the capture's warm-up iteration is part of the saved state): the
        # capture this run makes again must not train one more iteration
        self._capture_keeps_state = bool(tr["captured"])
        checkpoint.set_rng_state(tr["rng"], self.device)

    # ------------------------------------------------------------------ main.py:308-498
    def train(self) -> Tuple[float, Optional[Dict[str, object]]]:
        """The epoch loop.  On a Trainer restored by ``load`` it continues at the epoch after the saved one, with the saved
        best recall, early-stopping count and history."""
        args, data = self.args, self.data
        loop = self._resume or dict(epoch=0, best_recall=0.0, stopping_step=0, test_ret=None, history=[], stopped=False)
        self._resume = None
        stopping_step, best_recall, test_ret = loop["stopping_step"], loop["best_recall"], loop["test_ret"]
        self.history: List[Dict[str, float]] = list(loop["history"])
        ckpt_path = getattr(args, "checkpoint", "")     # a reference parse_args() Namespace has no such flag
        for epoch in range(loop["epoch"], 0 if loop["stopped"] else args.epoch):
            t1 = time()
            n_batch = data.n_train // args.batch_size + 1                                      # main.py:328
            acc = torch.zeros(4, dtype=torch.float32, device=self.device)                      # loss, mf, emb, cl
            self.step.start_epoch()
            for _ in range(n_batch):
                users, pos, neg = self.sample()
                if self.cuda_graph and self.step._graph is None and self.step.steady():
                    self.step.capture(keep_state=self._capture_keeps_state)
                out = self.step.step(users, pos, neg)
                acc[0] += out["batch_loss"].reshape(())
                acc[1:3] += out["loss5"][1:3]
                acc[3] += out["loss5"][4]
            loss, mf_loss, emb_loss, cl_loss = (float(v) for v in acc.cpu())                   # the epoch's only host read
            reg_loss = 0.0
            if math.isnan(loss):
                self.log("ERROR: loss is nan.")
                raise FloatingPointError("loss is nan")                                         # main.py:439-441 exits
            if (epoch + 1) % args.verbose != 0:
                # the reference prints its `contrastive_loss` variable here, which is initialised to 0. and never updated
                # (main.py:326, :443): the slot always reads 0.00000 -- kept for log parity; the accumulated value is in self.history
                self.log("Epoch %d [%.1fs]: train==[%.5f=%.5f + %.5f + %.5f  + %.5f]" % (epoch, time() - t1, loss, mf_loss, emb_loss,
                                                                                        reg_loss, 0.0))
                self.last_cl_loss = cl_loss
            t2 = time()
            stopped = False
            ret = self.test(list(data.val_set.keys()), is_val=True)                            # main.py:451-452 (every epoch)
            t3 = time()
            self.history.append(dict(epoch=epoch, loss=loss, mf_loss=mf_loss, emb_loss=emb_loss, recall=float(ret["recall"][1]),
                                     precision=float(ret["precision"][1]), ndcg=float(ret["ndcg"][1])))
            if args.verbose > 0:
                r, p, h, n = ret["recall"], ret["precision"], ret["hit_ratio"], ret["ndcg"]
                self.log("Epoch %d [%.1fs + %.1fs]: train==[%.5f=%.5f + %.5f + %.5f], recall=[%.5f, %.5f, %.5f, %.5f], "
                         "precision=[%.5f, %.5f, %.5f, %.5f], hit=[%.5f, %.5f, %.5f, %.5f], ndcg=[%.5f, %.5f, %.5f, %.5f]" %
                         (epoch, t2 - t1, t3 - t2, loss, mf_loss, emb_loss, reg_loss, r[0], r[1], r[2], r[-1], p[0], p[1], p[2], p[-1],
                          h[0], h[1], h[2], h[-1], n[0], n[1], n[2], n[-1]))
            if ret["recall"][1] > best_recall:                                                  # main.py:484-494
                best_recall = float(ret["recall"][1])
                test_ret = self.test(list(data.test_set.keys()), is_val=False)
                self.log("Test_Recall@%d: %.5f,  precision=[%.5f], ndcg=[%.5f]" % (self.Ks[1], test_ret["recall"][1],
                                                                                  test_ret["precision"][1], test_ret["ndcg"][1]))
                stopping_step = 0
            elif stopping_step < args.early_stopping_patience:
                stopping_step += 1
                self.log("#####Early stopping steps: %d #####" % stopping_step)
            else:
                self.log("#####Early stop! #####")
                stopped = True
            self._loop = dict(epoch=epoch + 1, best_recall=best_recall, stopping_step=stopping_step, test_ret=test_ret,
                              history=list(self.history), stopped=stopped)
            if ckpt_path:
                self.save(ckpt_path)
            if stopped:
                break
        self.log(str(test_ret))
        return best_recall, test_ret
