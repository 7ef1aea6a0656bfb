"""The whole hot step under the row-sharded scheme of north_star / SURVEY 8e: embedding tables, features and every
[U, d] / [I, d] intermediate are block-partitioned by rows over the ranks of one box, each rank holds the row blocks of the
normalised graphs (and of their transposes for the backward), and every SpMM is preceded by one all-gather of its dense
operand -- 2 per GCN layer forward, 2 backward, plus the modality / id propagations (parallel.RowShardedGCN is the same
schedule for the bare K-layer chain).  Everything else of the step is local to the rows a rank owns:

  projection + dropout   rows I_r of the features (no communication forward; dW, db all-reduced, they are [d, Dv+Dt])
  id fusion, layer mean, modality residual, softmax   row-wise
  losses                 the batch names rows of the FULL tables (main.py:368-370, :411-412).  Each rank contributes the
                         rows it owns (mmssl_gather_owned), ONE all-reduce of [5, B, d] gives every rank the batch rows
                         of u_f[users], i_f[pos], i_f[neg], Uvid[users], Utid[users]; the loss kernels then run replicated
                         (B = 1024: 0.27 GFLOP), and each rank keeps the gradient rows it owns (mmssl_scatter_add_owned) --
                         no second exchange, no cross-rank float atomics, bit-identical losses on every rank
  AdamW                  on the local row blocks of the two tables (optimiser state sharded with them); the five small
                         replicated parameters get identical all-reduced gradients and identical updates

The exchange is injected into ``Engine`` (``engine.exchange``): NCCL all-gather on the box, gloo in the CPU tests where the
kernels run under the emulator (tests/test_dist_emu.py).  Fusing the all-gather into the producing SpMM over NVSwitch
multicast (parallel.FusedRowShardedGCN) applies to the same call sites and is the next step for this class.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, checkpoint, ops
from ._lib import ptr, stream
from .engine import LIVE, P_EI, P_EU, Engine, FeatureStore, capture_graph
from .graph import SparseOperand
from .hotstep import HotStepConfig
from .parallel import RowPartition, all_gather_rows, shard_rows_scipy

REPLICATED = tuple(k for k in LIVE if k not in (P_EU, P_EI))


class RowBlockGraph:
    """What ``Engine`` needs of a graph, for one rank: ``fwd`` = A[rows_r, :] and ``bwd`` = (A^T)[cols_r, :] as prepared
    SpMM operands (global column ids), ``shape`` = the LOCAL (padded) row counts of the two row spaces, ``nnz`` = the
    global edge count (only compared with 0)."""

    def __init__(self, fwd: SparseOperand, bwd: SparseOperand, shape: Tuple[int, int], nnz: int,
                 fwd_part: Optional[SparseOperand] = None, bwd_part: Optional[SparseOperand] = None):
        self.fwd, self.bwd, self.shape, self.nnz = fwd, bwd, shape, int(nnz)
        # partial-product schedule: fwd_part = A[:, cols_r] (every row of A, the rank's columns, LOCAL column ids) so that
        # A @ X = sum over ranks of fwd_part_r @ X[cols_r];  bwd_part = (A^T)[:, rows_r] likewise for A^T @ dY
        self.fwd_part, self.bwd_part = fwd_part, bwd_part

    @classmethod
    def from_scipy(cls, mat, part_rows: RowPartition, part_cols: RowPartition, rank: int, device) -> "RowBlockGraph":
        def op(m, part):
            blk = shard_rows_scipy(m, part, rank).tocoo()
            t = lambda a, dt: torch.from_numpy(np.asarray(a).astype(dt)).to(device)
            o = SparseOperand(t(blk.row, "int64"), t(blk.col, "int64"), t(blk.data, "float32"), blk.shape[0], blk.shape[1])
            o.tighten()
            return o
        def col_block(m, part_r, part_c):
            """m[:, cols_r] with rows padded to world * block (the partial table's height) and local column ids."""
            lo, hi = part_c.bounds(rank)
            blk = m.tocsc()[:, lo:hi].tocoo()
            t = lambda a, dt: torch.from_numpy(np.asarray(a).astype(dt)).to(device)
            o = SparseOperand(t(blk.row, "int64"), t(blk.col, "int64"), t(blk.data, "float32"), part_r.world * part_r.block, part_c.block)
            o.tighten()
            return o
        mat = mat.tocsr()
        mt = mat.T.tocsr()
        return cls(op(mat, part_rows), op(mt, part_cols), (part_rows.block, part_cols.block), mat.nnz,
                   fwd_part=col_block(mat, part_rows, part_cols), bwd_part=col_block(mt, part_cols, part_rows))


    @classmethod
    def from_csr_blocks(cls, fwd_blk, bwd_blk, nnz: int, device, heights=None) -> "RowBlockGraph":
        """From two ``dataset.CsrBlock``s (the rank's rows of A and of A^T as ``ShardedDataset.operand`` maps them from disk:
        indptr rebased to 0, global column ids): a rank never sees the rest of the graph.  heights = (world * block of A's row
        space, world * block of its column space): padded heights of the two partial tables (default: the unpadded sizes)."""
        def op(blk):
            rows = np.repeat(np.arange(blk.shape[0], dtype=np.int64), np.diff(blk.indptr))
            t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).to(device)
            o = SparseOperand(t(rows, "int64"), t(blk.indices, "int64"), t(blk.values, "float32"), blk.shape[0], blk.shape[1])
            o.tighten()
            return o

        def transposed(blk, height):
            """(blk)^T with `height` (padded) rows: the column block of the other operand, local column ids."""
            rows = np.repeat(np.arange(blk.shape[0], dtype=np.int64), np.diff(blk.indptr))
            t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).to(device)
            o = SparseOperand(t(rows, "int64"), t(blk.indices, "int64"), t(blk.values, "float32"), blk.shape[0], height, transpose=True)
            o.tighten()
            return o
        h_rows, h_cols = heights if heights is not None else (bwd_blk.shape[1], fwd_blk.shape[1])
        return cls(op(fwd_blk), op(bwd_blk), (fwd_blk.shape[0], bwd_blk.shape[0]), nnz,
                   fwd_part=transposed(bwd_blk, h_rows), bwd_part=transposed(fwd_blk, h_cols))


def gather_owned(table: torch.Tensor, idx: torch.Tensor, lo: int, hi: int, out: torch.Tensor) -> torch.Tensor:
    lib = _lib.load(require_device=True)
    _lib.check(lib.mmssl_gather_owned(ptr(table), table.stride(0), ptr(idx), lo, hi, idx.numel(), table.shape[1], ptr(out),
                                      out.stride(0), stream()))
    return out


def scatter_add_owned(table: torch.Tensor, idx: torch.Tensor, lo: int, hi: int, src: torch.Tensor) -> None:
    lib = _lib.load(require_device=True)
    _lib.check(lib.mmssl_scatter_add_owned(ptr(table), table.stride(0), ptr(idx), lo, hi, idx.numel(), table.shape[1], ptr(src),
                                           src.stride(0), stream()))


def publish_rows(src: torch.Tensor, dst_local: torch.Tensor, y_mode: int = 0, y_raw: Optional[int] = None,
                 y_peers: Optional[Sequence[int]] = None) -> None:
    """mmssl_publish_rows: src -> the rank's row block of a (symmetric) table on every rank (see SymmetricTable.out_spec)."""
    import ctypes as C
    lib = _lib.load(require_device=True)
    peers = list(y_peers or [])
    arr = (C.c_void_p * max(len(peers), 1))(*peers)
    dst = C.c_void_p(int(y_raw)) if y_mode == 1 else ptr(dst_local)
    _lib.check(lib.mmssl_publish_rows(ptr(src), src.stride(0), src.shape[0], src.shape[1], dst, dst_local.stride(0), y_mode, len(peers), arr,
                                      stream()))


class MulticastExchange:
    """The exchange of the row-sharded step WITHOUT NCCL: every operand lives in a full-size table in CUDA symmetric memory
    (parallel.SymmetricTable, the class the fused SpMM + all-gather uses); a rank publishes its rows into every rank's copy with
    ONE kernel -- multimem.st through the NVSwitch multicast address, or peer stores when the allocation has no multicast
    address -- and ONE device-side signal-pad barrier orders producers and consumers.  Two tables per (row space, width) are
    used alternately: a table is overwritten only two exchanges later, i.e. after a barrier that every rank can only have
    reached once it had consumed the older contents.
    Tables are created lazily, in the (identical) order the ranks first need them: creation is a collective rendezvous."""

    def __init__(self, part_u: RowPartition, part_i: RowPartition, rank: int, device, group=None):
        self.parts = {"u": part_u, "i": part_i}
        self.rank, self.device, self.group = rank, device, group
        self.tabs: Dict[Tuple[str, int], list] = {}
        self.turn: Dict[Tuple[str, int], int] = {}

    def _table(self, space: str, width: int):
        from .parallel import SymmetricTable
        key = (space, width)
        if key not in self.tabs:
            self.tabs[key] = [SymmetricTable(self.parts[space], width, self.rank, self.device, self.group) for _ in range(2)]
            self.turn[key] = 0
        t = self.tabs[key][self.turn[key]]
        self.turn[key] ^= 1
        return t

    def gather(self, x: torch.Tensor, space: str) -> torch.Tensor:
        tab = self._table(space, x.shape[1])
        spec = tab.out_spec()
        publish_rows(x, tab.local_rows(), y_mode=spec["y_mode"], y_raw=spec["y_raw"][0] if "y_raw" in spec else None,
                     y_peers=spec["y_peers"][0] if "y_peers" in spec else None)
        tab.barrier()
        return tab.full()


class MulticastAllReduce:
    """Sum over the ranks of a flat fp32 buffer without NCCL: ``buffer`` (this rank's copy of a symmetric allocation) is where
    the contribution is written; ``reduce_into(out)`` = barrier, one kernel reading the sum through the multicast address
    (mmssl_mc_allreduce_sum), barrier.  Needs an NVSwitch multicast address (raises otherwise: the caller keeps NCCL then).
    ``ids=True``: an exact sum of ``numel`` int64 values instead -- ``write_ids(src)`` stores the contribution as four 16-bit limbs
    per value (mmssl_ids_to_limbs), ``reduce_into(out)`` reassembles the int64 sums (mmssl_mc_allreduce_ids)."""

    def __init__(self, numel: int, device, group=None, ids: bool = False):
        import torch.distributed._symmetric_memory as symm
        self.ids = ids
        n = 4 * numel if ids else (numel + 3) // 4 * 4
        g = group if group is not None else dist.group.WORLD
        self.buffer = symm.empty(n, dtype=torch.float32, device=device)
        self.buffer.zero_()
        self.h = symm.rendezvous(self.buffer, g.group_name)
        self.mc = int(self.h.multicast_ptr)
        if self.mc == 0:
            raise RuntimeError("NVSwitch multicast is not available for symmetric memory on this system")
        torch.cuda.synchronize(device)
        self.h.barrier()

    def write_ids(self, src: torch.Tensor) -> None:
        lib = _lib.load(require_device=True)
        assert self.ids and src.dtype == torch.int64 and src.is_contiguous() and 4 * src.numel() <= self.buffer.numel()
        _lib.check(lib.mmssl_ids_to_limbs(ptr(src), ptr(self.buffer), src.numel(), stream()))

    def reduce_into(self, out: torch.Tensor) -> torch.Tensor:
        import ctypes as C
        lib = _lib.load(require_device=True)
        assert out.is_contiguous()
        self.h.barrier()                         # every rank's contribution is in its copy
        if self.ids:
            assert out.dtype == torch.int64 and 4 * out.numel() <= self.buffer.numel()
            _lib.check(lib.mmssl_mc_allreduce_ids(C.c_void_p(self.mc), ptr(out), out.numel(), stream()))
        else:
            assert out.numel() % 4 == 0 and out.numel() <= self.buffer.numel()
            _lib.check(lib.mmssl_mc_allreduce_sum(C.c_void_p(self.mc), ptr(out), out.numel(), stream()))
        self.h.barrier()                         # every rank has read: the buffer may be rewritten
        return out


class PartialTables:
    """Full-height partial-product tables of the "reduce_scatter" schedule, in CUDA symmetric memory: every rank writes
    A[:, cols_r] @ X[cols_r] into its own copy, one signal-pad barrier, then each rank reads the rows it owns of the SUM over the
    copies through the multicast address (mmssl_reduce_rows_epilogue: multimem.ld_reduce + the SpMM epilogue).  Two tables per
    width are used alternately: a table is rewritten only two exchanges later, after a barrier every rank can only have
    reached once it had read the older contents.  Created lazily, in the (identical) order the ranks first need them."""

    def __init__(self, part: RowPartition, rank: int, device, group=None):
        self.part, self.rank, self.device, self.group = part, rank, device, group
        self.tabs: Dict[int, list] = {}
        self.turn: Dict[int, int] = {}

    def next(self, width: int):
        import torch.distributed._symmetric_memory as symm
        if width not in self.tabs:
            g = self.group if self.group is not None else dist.group.WORLD
            pair = []
            for _ in range(2):
                t = symm.empty(self.part.world * self.part.block, width, dtype=torch.float32, device=self.device)
                t.zero_()
                h = symm.rendezvous(t, g.group_name)
                mc = int(h.multicast_ptr)
                if mc == 0:
                    raise RuntimeError("NVSwitch multicast is not available for symmetric memory on this system")
                pair.append((t, h, mc))
            torch.cuda.synchronize(self.device)
            pair[0][1].barrier()
            self.tabs[width], self.turn[width] = pair, 0
        t = self.tabs[width][self.turn[width]]
        self.turn[width] ^= 1
        return t


def reduce_rows_epilogue(srcs, n_rows: int, d: int, ys, *, multicast: bool, epilogue=0, alpha=1.0, cs=None, ysaved=None, ss=None,
                         s_mode=0, sbases=None):
    """mmssl_reduce_rows_epilogue: srcs[r] = raw address (multicast) or tensor (reduced rows) of the rank's rows, right-hand side r."""
    import ctypes as C
    from ._lib import SpmmRhs
    lib = _lib.load(require_device=True)
    nrhs = len(ys)
    rhs = (SpmmRhs * nrhs)()
    ld_ = lambda t: 0 if t is None else int(t.stride(0))
    for r in range(nrhs):
        c = cs[r] if cs is not None else None
        yv = ysaved[r] if ysaved is not None else None
        sr = ss[r] if ss is not None else None
        sb = sbases[r] if sbases is not None else None
        src, lds_ = srcs[r]
        rhs[r] = SpmmRhs(C.c_void_p(int(src)), int(lds_), ptr(ys[r]), ld_(ys[r]), ptr(c), ld_(c), ptr(yv), ld_(yv), ptr(sr), ld_(sr),
                         ptr(sb), ld_(sb))
    _lib.check(lib.mmssl_reduce_rows_epilogue(n_rows, d, nrhs, rhs, epilogue, float(alpha), s_mode, 1 if multicast else 0, stream()))
    return list(ys)


class RowShardedHotStep:
    """One rank of the row-sharded hot step.  ``params``: the rank's padded row blocks of the two embedding tables
    (``RowPartition.local``) and full copies of the five small parameters; ``feats``: FeatureStores of the rank's item rows;
    ``graphs``: six RowBlockGraphs (ui, iu, image ui/iu, text ui/iu; pass the same objects to alias them, main.py:68-69)."""

    def __init__(self, params: Dict[str, torch.Tensor], feats: Sequence[FeatureStore], graphs: Sequence[RowBlockGraph],
                 cfg: HotStepConfig, batch: int, part_u: RowPartition, part_i: RowPartition, rank: int, group=None,
                 optimizer_step: bool = True, exchange: str = "nccl", schedule: str = "reduce_scatter", sampler=None):
        self.cfg, self.batch, self.pu, self.pi, self.rank, self.group = cfg, batch, part_u, part_i, rank, group
        # optional sampler.ShardedTripleSampler: every run() draws the batch of (seed, step_dev) on the device, so every replay of
        # a captured step trains on a fresh batch; without it the batch is what set_indices wrote
        self.sampler = sampler
        if sampler is not None:
            sampler.reserve(batch)
        self.P = {k: params[k] for k in LIVE}
        self.feats, self.graphs = tuple(feats), tuple(graphs)
        self.engine = Engine(cfg.embed_size, cfg.n_layers, cfg.head_num, cfg.id_cat_rate, cfg.model_cat_rate, cfg.proj_impl)
        # NCCL / gloo collectives order the work on one stream.  With the multicast exchange every exchange is a kernel plus a
        # device-side signal-pad barrier on its own symmetric table, so the modality branch (tables of width 2d) and the id / GCN
        # branch (width d) can overlap one branch's exchange with the other's SpMMs, like on one GPU (engine.two_streams).
        import os as _os
        self.engine.two_streams = (exchange == "multicast" and part_u.world > 1 and _os.environ.get("MMSSL_ROWSHARD_STREAMS", "1") == "1")
        self.engine.exchange = self._exchange
        # schedule of the products whose dense operand lives in the user space (A_iu @ u, A_ui^T @ du, ...):
        #   "allgather"      all-gather the user-sized operand, multiply the rank's rows (round 1)
        #   "reduce_scatter" multiply the rank's COLUMN block, reduce-scatter the item-sized result (only the smaller, item-side
        #                    table ever crosses NVLink: syn1m 0.1 GB instead of 0.5 GB per exchange)
        if schedule not in ("allgather", "reduce_scatter"):
            raise ValueError("schedule must be 'allgather' or 'reduce_scatter'")
        self.schedule = schedule if part_u.world > 1 and all(g.fwd_part is not None for g in graphs) else "allgather"
        self.engine.sharded_spmm = self._sharded_spmm
        self.partials = None
        # "nccl": all_gather_into_tensor (gloo in the CPU tests); "multicast": MulticastExchange (symmetric memory, no NCCL)
        self.mc = MulticastExchange(part_u, part_i, rank, self.P[P_EU].device, group) if exchange == "multicast" and part_u.world > 1 else None
        if exchange not in ("nccl", "multicast"):
            raise ValueError("exchange must be 'nccl' or 'multicast'")
        self.optimizer_step = optimizer_step
        self.n_gathers, self.gathered_bytes = 0, 0
        self.n_reduce_scatters = 0
        dev = self.P[P_EU].device
        d, B = cfg.embed_size, batch
        f = dict(dtype=torch.float32, device=dev)
        self.idx = torch.zeros(3, B, dtype=torch.int64, device=dev)
        self.rows = torch.zeros(5, B, d, **f)               # u_f[users], i_f[pos], i_f[neg], Uvid[users], Utid[users]
        self.rows_part = self.rows                          # where the rank's contribution is written (== rows with NCCL: in place)
        self.ar_rows = self.ar_flat = None
        self.g_rows = torch.zeros(5, B, d, **f)
        self.g_uf = torch.zeros(part_u.block, d, **f)
        self.g_if = torch.zeros(part_i.block, d, **f)
        self.g_uvid = torch.zeros(part_u.block, d, **f)
        self.g_utid = torch.zeros(part_u.block, d, **f)
        # image and text graphs are the same object at step 0 (main.py:68-69): Uvid is Utid, one InfoNCE counted twice
        self.alias = graphs[2] is graphs[4] and graphs[3] is graphs[5]
        self.nce = [ops.InfoNCEWork(B, d, dev) for _ in range(1 if self.alias else 2)]
        self.cl_seed = torch.full((1,), cfg.cl_rate * (2.0 if self.alias else 1.0), **f)
        self.out5 = torch.zeros(5, **f)
        self.grads = {k: torch.zeros_like(t) for k, t in self.P.items()}
        self.m = {k: torch.zeros_like(t) for k, t in self.P.items()}
        self.v = {k: torch.zeros_like(t) for k, t in self.P.items()}
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.masks: Optional[tuple] = None                  # injected [I_block, d] keep-masks of the rank's item rows
        self.training = True
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        # the small replicated gradients travel in one flat buffer
        n = sum((self.grads[k].numel() + 3) // 4 * 4 for k in REPLICATED) + 4      # + one slot for the local feat_reg term
        self._feat_slot = n - 4
        self._flat = torch.zeros(n, **f)
        self._flat_part = self._flat
        if self.mc is not None:                             # all-reduce through multimem.ld_reduce instead of NCCL, when there is multicast
            try:
                self.ar_rows = MulticastAllReduce(5 * B * d, dev, group)
                self.ar_flat = MulticastAllReduce(n, dev, group)
                self.rows_part = self.ar_rows.buffer[:5 * B * d].view(5, B, d)
                self._flat_part = self.ar_flat.buffer[:n]
            except RuntimeError:
                self.ar_rows = self.ar_flat = None
        # Engine.backward writes the small gradients into views of the contribution buffer; AdamW reads views of the reduced one
        self.grads_part = dict(self.grads)
        o = 0
        for k in REPLICATED:
            g = self.grads[k]
            self.grads_part[k] = self._flat_part[o:o + g.numel()].view_as(g)
            self.grads[k] = self._flat[o:o + g.numel()].view_as(g)
            o += (g.numel() + 3) // 4 * 4

    # -------------------------------------------------------------- exchange
    def _exchange(self, xs: List[torch.Tensor], space: str) -> List[torch.Tensor]:
        part = self.pu if space == "u" else self.pi
        if len(xs) == 2 and xs[0].stride() == xs[1].stride() and xs[0].shape == xs[1].shape and xs[0].stride(1) == 1 and \
                xs[0].stride(0) == 2 * xs[0].shape[1] and xs[1].data_ptr() == xs[0].data_ptr() + 4 * xs[0].shape[1]:
            # image | text halves of one [rows, 2d] buffer (engine.X2 / U2 / I2 and their gradients): one collective
            w = xs[0].shape[1]
            both = self._exchange([torch.as_strided(xs[0], (xs[0].shape[0], 2 * w), (2 * w, 1))], space)[0]
            return [both[:, :w], both[:, w:]]
        out = []
        for x in xs:
            self.n_gathers += 1
            self.gathered_bytes += x.numel() * x.element_size() * (part.world - 1)
            out.append(self.mc.gather(x.contiguous(), space) if self.mc is not None else all_gather_rows(x, part, self.group))
        return out

    def _sharded_spmm(self, g, which: str, xs, space: str, ys=None, **kw):
        """Engine hook: Y = epi(op(g) @ X) with X a row block of a table that lives in `space`."""
        if space == "i" or self.schedule == "allgather":
            return ops.spmm(getattr(g, which), self._exchange(list(xs), space), ys, **kw)
        # the operand is user-sized: partial product over the rank's columns into full-height item-space tables, then the
        # rank's rows of the sum over ranks + the epilogue the SpMM would have applied
        op = g.fwd_part if which == "fwd" else g.bwd_part
        d = xs[0].shape[1]
        nrhs = len(xs)
        part = self.pi
        lo = self.rank * part.block
        if ys is None:
            ys = [torch.empty(part.block, d, dtype=torch.float32, device=xs[0].device) for _ in range(nrhs)]
        self.n_reduce_scatters += 1
        self.gathered_bytes += part.block * d * nrhs * 4 * (part.world - 1)
        if self.mc is not None:
            if self.partials is None:
                self.partials = PartialTables(part, self.rank, xs[0].device, self.group)
            tab, h, mc = self.partials.next(nrhs * d)
            outs = [tab[:, r * d:(r + 1) * d] for r in range(nrhs)]
            ops.spmm(op, [x if x.stride(1) == 1 else x.contiguous() for x in xs], outs)
            h.barrier()                                             # every rank's partial table is complete
            srcs = [(mc + (lo * nrhs * d + r * d) * 4, nrhs * d) for r in range(nrhs)]
            return reduce_rows_epilogue(srcs, part.block, d, ys, multicast=True, **kw)
        full = torch.empty(part.world * part.block, nrhs * d, dtype=torch.float32, device=xs[0].device)
        outs = [full[:, r * d:(r + 1) * d] for r in range(nrhs)]
        ops.spmm(op, [x if x.stride(1) == 1 else x.contiguous() for x in xs], outs)
        if dist.get_backend(self.group) == "gloo":                  # CPU tests: gloo has no reduce-scatter
            dist.all_reduce(full, op=dist.ReduceOp.SUM, group=self.group)
            mine = full[lo:lo + part.block]
        else:
            mine = torch.empty(part.block, nrhs * d, dtype=torch.float32, device=xs[0].device)
            dist.reduce_scatter_tensor(mine, full, op=dist.ReduceOp.SUM, group=self.group)
        srcs = [(mine[:, r * d:(r + 1) * d].data_ptr(), nrhs * d) for r in range(nrhs)]
        self._keep = mine
        return reduce_rows_epilogue(srcs, part.block, d, ys, multicast=False, **kw)

    def _masks(self):
        if not self.training or self.cfg.drop_rate <= 0:
            return None
        if self.masks is not None:
            return self.masks
        import torch.nn.functional as F
        ones = torch.ones(self.pi.block, self.cfg.embed_size, dtype=torch.float32, device=self.idx.device)
        return (F.dropout(ones, self.cfg.drop_rate, True), F.dropout(ones, self.cfg.drop_rate, True))

    def set_indices(self, users, pos, neg) -> None:
        for j, t in enumerate((users, pos, neg)):
            self.idx[j].copy_(torch.as_tensor(t, dtype=torch.int64), non_blocking=True)

    # -------------------------------------------------------------- one step
    def run(self) -> torch.Tensor:
        """One hot step on the batch in ``self.idx`` (GLOBAL user / item ids, identical on every rank; drawn into it first when
        the step has a sampler).  Returns the device
        tensor [total, mf, emb, feat_reg, cl] -- global values, identical on every rank."""
        cfg, B = self.cfg, self.batch
        users, pos, neg = self.idx[0], self.idx[1], self.idx[2]
        ulo, uhi = self.pu.bounds(self.rank)
        ilo, ihi = self.pi.bounds(self.rank)
        for t in (self.g_uf, self.g_if, self.g_uvid, self.g_utid, self.g_rows):
            t.zero_()
        outs, st = self.engine.forward(self.P, self.feats, self.graphs, self._masks(), want_sumsq=True)
        u_f, i_f, _, _, _, _, u_vid, u_tid, _, _ = outs
        alias = self.alias
        if self.sampler is not None:                        # (seed, optimiser step) -> the batch, identical on every rank
            self.sampler.sample_into(self.idx, step_dev=self.step_dev)
        # ---- the batch rows of the full tables: owned rows + one all-reduce
        part = self.rows_part
        gather_owned(u_f, users, ulo, uhi, part[0])
        gather_owned(i_f, pos, ilo, ihi, part[1])
        gather_owned(i_f, neg, ilo, ihi, part[2])
        gather_owned(u_vid, users, ulo, uhi, part[3])
        if not alias:
            gather_owned(u_tid, users, ulo, uhi, part[4])
        if self.ar_rows is not None:
            self.ar_rows.reduce_into(self.rows)
        elif self.pu.world > 1:
            dist.all_reduce(self.rows, op=dist.ReduceOp.SUM, group=self.group)
        ub, pb, nb, zv, zt = self.rows
        g_ub, g_pb, g_nb, g_zv, g_zt = self.g_rows
        # ---- losses on the compact batch tables (identity indices), replicated on every rank
        reg_coef = cfg.emb_decay / cfg.batch_size
        bpr_part, n_bpr = ops.bpr(ub, pb, nb, None, None, None, mode=3, reg_coef=reg_coef, g_u=g_ub, g_p=g_pb, g_n=g_nb)
        inv_tau = 1.0 / cfg.tau
        parts = []
        for w, z1, gz1 in zip(self.nce, (zv, zt), (g_zv, g_zt)):
            parts.append(ops.infonce_forward(z1, ub, None, inv_tau, w, g_loss=self.cl_seed))
            if st.fused:
                ops.infonce_backward(None, inv_tau, w, gz1, g_ub)
        nce1, nce2 = parts[0], parts[-1]
        ops.loss_assemble(bpr_part, n_bpr, B, reg_coef, st.sumsq_u, st.sumsq_i, 0.5 * cfg.feat_reg_decay / self.pi.n, nce1, nce2, B,
                          cfg.cl_rate, self.out5)
        # ---- gradient rows go back to their owners
        scatter_add_owned(self.g_uf, users, ulo, uhi, g_ub)
        scatter_add_owned(self.g_if, pos, ilo, ihi, g_pb)
        scatter_add_owned(self.g_if, neg, ilo, ihi, g_nb)
        if st.fused:
            scatter_add_owned(self.g_uvid, users, ulo, uhi, g_zv)
            if not alias:
                scatter_add_owned(self.g_utid, users, ulo, uhi, g_zt)
        grads = [self.g_uf, self.g_if, None, None, None, None, self.g_uvid if st.fused else None,
                 (None if alias else self.g_utid) if st.fused else None, None, None]
        self.engine.backward(st, self.P, self.feats, grads, feat_reg_coef=cfg.feat_reg_decay / self.pi.n, out=self.grads_part)
        self._flat_part[self._feat_slot:self._feat_slot + 1] = self.out5[3:4]       # feat_reg was summed over the local rows only:
                                                                                    # it rides along with the small gradients
        for k in (P_EU, P_EI):                              # the table gradients are private to the rank (same tensors in both dicts)
            self.grads[k] = self.grads_part[k]
        if self.ar_flat is not None:                        # dW, db, dWcat: sums over the ranks' rows
            self.ar_flat.reduce_into(self._flat)
        elif self.pu.world > 1:
            dist.all_reduce(self._flat, op=dist.ReduceOp.SUM, group=self.group)
        if self.pu.world > 1:
            # the total is formed again from the all-reduced feat_reg, in loss_assemble's order, from terms that are equal on
            # every rank: `total += feat - feat_local` rounded differently on each rank, and the losses differed in the last bit
            self.out5[3] = self._flat[self._feat_slot]
            self.out5[0] = self.out5[1] + self.out5[2] + self.out5[3] + cfg.cl_rate * self.out5[4]
        if self.optimizer_step:
            ops.step_tick(self.step_dev)
            keys = list(LIVE)
            ops.adamw([self.P[k] for k in keys], [self.grads[k] for k in keys], [self.m[k] for k in keys], [self.v[k] for k in keys],
                      self.step_dev, cfg.lr, cfg.beta1, cfg.beta2, cfg.eps, cfg.weight_decay)
        return self.out5

    # -------------------------------------------------------------- evaluation
    def _quiesce(self) -> None:
        """With the multicast exchange a rank publishes into the symmetric tables of EVERY rank, and the captured step uses the
        same tables: wait until no rank is inside a step or an exchange."""
        if self.mc is not None:
            torch.cuda.synchronize(self.idx.device)
            dist.barrier(group=self.group)

    def final_embeddings(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """Collective.  The model's eval-mode forward (no dropout, no losses, no optimiser step) through the step's own exchange:
        the rank's padded [block, d] rows of the final user and item tables (u_f, i_f), fresh tensors.  Writes nothing a later
        step or a captured step reads: the forward allocates its outputs, and what it shares with the step -- the SpMM split-row
        partials and the multicast exchange tables -- is scratch that every step writes before it reads (the barriers around
        keep the ranks out of each other's exchanges).  The exchange counters keep counting training steps only."""
        counters = (self.n_gathers, self.gathered_bytes, self.n_reduce_scatters)
        self._quiesce()
        outs, _ = self.engine.forward(self.P, self.feats, self.graphs, None, want_sumsq=False)
        self._quiesce()
        self.n_gathers, self.gathered_bytes, self.n_reduce_scatters = counters
        return outs[0], outs[1]

    def test(self, evaluator, users_to_test, is_val: bool) -> Dict[str, object]:
        """Collective.  ``Trainer.test`` of the row-sharded model: ``evaluator`` is this rank's ``evaluate.ShardedEvaluator``;
        returns its ``test_torch`` result, identical on every rank."""
        u_f, i_f = self.final_embeddings()
        return evaluator.test_torch(u_f, i_f, users_to_test, is_val)

    # -------------------------------------------------------------- checkpoint (checkpoint.py)
    def meta(self) -> dict:
        """Same fields as HotStep.meta; the training-matrix fingerprint is summed over the ranks' row blocks (a collective on the
        first call; the training graph never changes, so it is kept)."""
        if self._fingerprint is None:
            ulo, _ = self.pu.bounds(self.rank)
            nnz, h = checkpoint.graph_fingerprint(self.graphs[0], row0=ulo)
            if self.pu.world > 1:    # 16-bit limbs: the sum over the ranks cannot overflow int64; recombined mod 2^64 below
                t = torch.tensor([(h >> (16 * j)) & 0xFFFF for j in range(4)] + [nnz], dtype=torch.int64, device=self.idx.device)
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
                v = [int(x) for x in t.cpu()]
                h, nnz = sum(v[j] << (16 * j) for j in range(4)) & ((1 << 64) - 1), v[4]
            self._fingerprint = (nnz, h)
        m = checkpoint.make_meta(self.pu.n, self.pi.n, self.cfg, self.batch, self.feats, self._fingerprint)
        if self.sampler is not None:         # the batch of (seed, step) does not depend on the world size
            m["sampler_seed"] = int(self.sampler.seed)
        return m

    _fingerprint = None

    def state_dict(self) -> dict:
        """This rank's file of a row-sharded checkpoint (every rank calls it: the fingerprint is a collective): the REAL rows of
        the rank's blocks of the two tables and of their moments (padding dropped, global row ranges in ``rows``); rank 0 also
        holds the replicated parameters, their moments and the step counter."""
        (ulo, uhi), (ilo, ihi) = self.pu.bounds(self.rank), self.pi.bounds(self.rank)
        rows = {P_EU: uhi - ulo, P_EI: ihi - ilo}
        keys = [k for k in LIVE if k in rows or self.rank == 0]
        pick = lambda d: {k: (d[k][:rows[k]] if k in rows else d[k]) for k in keys}
        return dict(format=checkpoint.FORMAT, kind="rowshard", meta=self.meta(), rows={"user": (ulo, uhi), "item": (ilo, ihi)},
                    model=pick(self.P), optim=dict(m=pick(self.m), v=pick(self.v), step=int(self.step_dev.cpu()[0])))

    def load_state_dict(self, state: dict) -> None:
        """Copies ``checkpoint.read_sharded(directory, world, rank)`` of this rank into the live buffers in place."""
        checkpoint.check_format(state, ("rowshard", "hotstep"))
        checkpoint.check_meta(state["meta"], self.meta())
        want = {"user": self.pu.bounds(self.rank), "item": self.pi.bounds(self.rank)}
        if {k: tuple(v) for k, v in state.get("rows", want).items()} != want:
            raise ValueError(f"checkpoint mismatch in rows: saved {state['rows']}, this rank {want}")
        checkpoint.copy_into(self.P, state["model"], "model")
        checkpoint.copy_into(self.m, state["optim"]["m"], "optim.m")
        checkpoint.copy_into(self.v, state["optim"]["v"], "optim.v")
        self.step_dev.fill_(int(state["optim"]["step"]))

    def save(self, directory: str) -> None:
        """Collective: every rank writes its file of the checkpoint into ``directory``."""
        checkpoint.save_sharded(self, directory)

    def load(self, directory: str) -> None:
        """Collective: every rank reads the rows of its blocks from a checkpoint written at any world size."""
        self.load_state_dict(checkpoint.read_sharded(directory, self.pu.world, self.rank))

    # -------------------------------------------------------------- CUDA graph
    def capture(self, warmup: int = 2) -> None:
        """Capture ``run`` into a CUDA graph (static buffers; update the indices with ``set_indices`` between replays, or give the
        step a sampler: each replay then draws the batch of its step).  Only with the
        multicast exchange or a single rank: every exchange is then a kernel plus a device-side signal-pad barrier, which a graph
        can hold; NCCL collectives inside a capture hung in round 1 and are refused here.  EXPERIMENTAL until its first GPU run."""
        if self.pu.world > 1 and self.mc is None:
            raise RuntimeError("capture() needs exchange='multicast' (NCCL collectives are not captured)")
        if self.pu.world > 1 and self.ar_rows is None:
            raise RuntimeError("capture() needs the multicast all-reduce (no NVSwitch multicast address on this system)")
        if self.sampler is not None and self.sampler.exchange is not None and self.sampler.ar.get(self.batch) is None:
            raise RuntimeError("capture() needs a sampler with exchange='multicast' (its NCCL all-reduce is not captured)")

        def warm():
            for _ in range(warmup):
                self.run()
        self._graph, _ = capture_graph(warm, self.run)

    def replay(self) -> torch.Tensor:
        if self._graph is None:
            raise RuntimeError("call capture() first")
        self._graph.replay()
        return self.out5


def shard_problem(P_full: Dict[str, torch.Tensor], feats_full: Sequence[torch.Tensor], ui_norm, iu_norm, rank: int, world: int, device):
    """Rank-local pieces of a full problem: (params, FeatureStores, six RowBlockGraphs with the modality graphs aliased,
    part_u, part_i).  The full problem only has to exist on the host."""
    U, I = ui_norm.shape
    pu, pi = RowPartition(U, world), RowPartition(I, world)
    P = {k: P_full[k].to(device).clone().contiguous() for k in REPLICATED}      # private copies: the step updates them in place
    P[P_EU] = pu.local(P_full[P_EU], rank).to(device).contiguous()
    P[P_EI] = pi.local(P_full[P_EI], rank).to(device).contiguous()
    feats = tuple(FeatureStore(pi.local(f, rank).to(device).contiguous(), keep_fp32=True) for f in feats_full)
    g_ui = RowBlockGraph.from_scipy(ui_norm, pu, pi, rank, device)
    g_iu = RowBlockGraph.from_scipy(iu_norm, pi, pu, rank, device)
    return P, feats, (g_ui, g_iu, g_ui, g_iu, g_ui, g_iu), pu, pi


def shard_problem_from_disk(root: str, P_full: Dict[str, torch.Tensor], rank: int, world: int, device):
    """Same pieces as ``shard_problem`` but read from a shard directory written once by ``dataset.write_shards`` (SURVEY 8f #4):
    every rank memory-maps only its row blocks of the four operands and its item rows of the two feature matrices."""
    from .dataset import ShardedDataset
    sh = ShardedDataset.open(root, rank, world)
    pu, pi = sh.part["user"], sh.part["item"]
    P = {k: P_full[k].to(device).clone().contiguous() for k in REPLICATED}      # private copies: the step updates them in place
    P[P_EU] = pu.local(P_full[P_EU], rank).to(device).contiguous()
    P[P_EI] = pi.local(P_full[P_EI], rank).to(device).contiguous()
    feats = []
    for which in ("image", "text"):
        f = torch.zeros(pi.block, sh.meta[f"{which}_dim"], dtype=torch.float32)
        rows = sh.features(which)
        f[:rows.shape[0]] = torch.from_numpy(np.ascontiguousarray(rows))
        feats.append(FeatureStore(f.to(device), keep_fp32=True))
    nnz = sh.meta["operands"]["ui"]["nnz"]
    hu, hi_ = pu.world * pu.block, pi.world * pi.block
    g_ui = RowBlockGraph.from_csr_blocks(sh.operand("ui"), sh.operand("uiT"), nnz, device, heights=(hu, hi_))
    g_iu = RowBlockGraph.from_csr_blocks(sh.operand("iu"), sh.operand("iuT"), nnz, device, heights=(hi_, hu))
    return P, tuple(feats), (g_ui, g_iu, g_ui, g_iu, g_ui, g_iu), pu, pi
