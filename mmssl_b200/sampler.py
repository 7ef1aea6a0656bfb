"""Device-side triple sampler (SURVEY 8f "next" #1): the reference's ``Data.sample``
(utility/load_data.py:153-191) as CUDA kernels, so a training step needs no host input at all.
Batches of up to 1024 triples take one single-CTA launch; larger batches take an exact multi-CTA
radix select over all users that have a training item (csrc/sampler.cu).

``ShardedTripleSampler`` draws the same batches when every rank holds only the training rows of its own block of users (a
row-sharded run): the slot selection depends on (seed, step, batch, n_exist) alone and is replicated on every rank, the rank
that owns a slot's user draws its positive and negative, and one exact integer sum over the ranks gives every rank the batch.
At any world size the batch at (seed, step, B) is bitwise ``DeviceTripleSampler(R, seed).sample_into(out, step=step)`` on the
whole training matrix R."""
from __future__ import annotations

import numpy as np
import torch

import torch.distributed as dist

from . import _lib
from ._lib import ptr, stream

ONE_CTA_MAX_BATCH = 1024


class DeviceTripleSampler:
    def __init__(self, train_csr, device="cuda", seed: int = 2022):
        lib = _lib.load(require_device=True)
        csr = train_csr.tocsr()
        csr.sort_indices()
        self.n_users, self.n_items = csr.shape
        self.indptr = torch.from_numpy(csr.indptr.astype(np.int64)).to(device)
        self.indices = torch.from_numpy(csr.indices.astype(np.int64)).to(device)
        exist = np.nonzero(np.diff(csr.indptr) > 0)[0].astype(np.int64)
        self.exist = torch.from_numpy(exist).to(device)
        self.claim = torch.empty(max(len(exist), 1), dtype=torch.int32, device=device)
        self.seed = seed
        self.device = device
        self.ws = {}            # batch size -> workspace of the multi-CTA path
        _lib.check(lib.mmssl_sampler_init(ptr(self.claim), len(exist), stream()))

    def reserve(self, batch: int) -> None:
        """Allocates the multi-CTA workspace of `batch` (batch > 1024) up front, e.g. before a CUDA-graph capture.
        The workspace carries the select's counters from kernel to kernel, so calls of one sampler with the same batch size
        must not run concurrently (two streams, or two graphs replayed at once); give concurrent callers a sampler each."""
        if batch <= ONE_CTA_MAX_BATCH or batch in self.ws:
            return
        lib = _lib.load(require_device=True)
        nbytes = lib.mmssl_sampler_workspace_bytes(self.exist.numel(), batch)
        if nbytes < 0:
            raise _lib.MmsslLibraryError("mmssl_sampler_workspace_bytes failed")
        # zero-filled once: the select's counters start at zero and every call leaves them so
        self.ws[batch] = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device=self.device)

    def sample_into(self, out: torch.Tensor, step_dev: torch.Tensor = None, step: int = 0) -> torch.Tensor:
        """Fills out[3, B] (int64: users, pos, neg).  `step_dev` (int32 device scalar) makes the launch
        replayable inside a CUDA graph with a fresh batch per replay."""
        lib = _lib.load(require_device=True)
        assert out.dtype == torch.int64 and out.dim() == 2 and out.shape[0] == 3 and out.is_contiguous()
        b = out.shape[1]
        if b <= ONE_CTA_MAX_BATCH:
            _lib.check(lib.mmssl_sample_triples(ptr(self.indptr), ptr(self.indices), ptr(self.exist), self.exist.numel(),
                                                self.n_items, b, self.seed, ptr(step_dev), int(step), ptr(self.claim),
                                                ptr(out[0]), ptr(out[1]), ptr(out[2]), stream()))
            return out
        self.reserve(b)
        ws = self.ws[b]
        _lib.check(lib.mmssl_sample_triples_multi(ptr(self.indptr), ptr(self.indices), ptr(self.exist), self.exist.numel(),
                                                  self.n_items, b, self.seed, ptr(step_dev), int(step), ptr(ws), ws.numel(),
                                                  ptr(out[0]), ptr(out[1]), ptr(out[2]), stream()))
        return out


class ShardedTripleSampler:
    """One rank's part of the device sampler of a row-sharded run.  ``rows``: the rank's training rows (``dataset.CsrBlock`` of
    the user block ``part_u.bounds(rank)``: indptr rebased to 0, sorted GLOBAL item ids; ``ShardedDataset.train_rows()``; its
    arrays may be numpy or device tensors).
    Construction is a collective over ``group`` (one all-gather of the per-rank counts of non-empty rows).  The slots of the
    one-GPU sampler are the non-empty rows in ascending global user id; rank r owns the slots [off[r], off[r] + count[r]).
    ``exchange``: "nccl" sums the ranks' [3, B] int64 outputs with one ``dist.all_reduce`` (gloo in the CPU tests); "multicast"
    exactly through the NVSwitch multicast address of a symmetric buffer (each id as four 16-bit limbs summed by
    multimem.ld_reduce.add.v4.f32, exact) between two signal-pad barriers, which a CUDA graph can hold (rowshard_step.MulticastAllReduce; NCCL when the system has no multicast).
    The claim table / select workspace are sized for the GLOBAL n_exist on every rank."""

    def __init__(self, rows, part_u, rank: int, group=None, device="cuda", seed: int = 2022, exchange: str = "nccl"):
        lib = _lib.load(require_device=True)
        if exchange not in ("nccl", "multicast"):
            raise ValueError("exchange must be 'nccl' or 'multicast'")
        lo, hi = part_u.bounds(rank)
        if (rows.lo, rows.hi) != (lo, hi):
            raise ValueError(f"rows [{rows.lo}, {rows.hi}) are not the user block [{lo}, {hi}) of rank {rank}")
        self.part_u, self.rank, self.group, self.seed, self.device = part_u, rank, group, seed, device
        self.n_users, self.n_items = part_u.n, int(rows.shape[1])
        def dev(a, dtype):          # numpy (a memory map of ShardedDataset) or a tensor already on the device
            t = a if torch.is_tensor(a) else torch.from_numpy(np.array(a))
            return t.to(device=device, dtype=dtype).contiguous()
        self.row0 = lo
        self.indptr = dev(rows.indptr, torch.int64)[:hi - lo + 1]
        self.indices = dev(rows.indices, torch.int32)
        self.exist = torch.nonzero(self.indptr[1:] > self.indptr[:-1]).flatten()      # local rows, ascending
        n_local = self.exist.numel()
        counts = [n_local] * part_u.world
        if part_u.world > 1:
            mine = torch.tensor([n_local], dtype=torch.int64, device=device)
            got = [torch.zeros_like(mine) for _ in range(part_u.world)]
            dist.all_gather(got, mine, group=group)
            counts = [int(t.cpu()[0]) for t in got]
        self.n_exist = sum(counts)
        if self.n_exist == 0:
            raise ValueError("no user has a training item")
        self.slot_lo = sum(counts[:rank])
        self.slot_hi = self.slot_lo + n_local
        self.claim = torch.empty(self.n_exist, dtype=torch.int32, device=device)
        self.ws = {}            # batch size -> workspace of the multi-CTA path
        self.ar = {}            # batch size -> MulticastAllReduce of the [3, B] batch
        self.own = {}           # batch size -> this rank's [3, B] contribution (multicast exchange)
        self.exchange = exchange if part_u.world > 1 else None
        _lib.check(lib.mmssl_sampler_init(ptr(self.claim), self.n_exist, stream()))

    def reserve(self, batch: int) -> None:
        """Allocates what a batch of this size needs up front (before a CUDA-graph capture): the multi-CTA workspace and, with the
        multicast exchange, the symmetric buffer (a collective).  As for ``DeviceTripleSampler``, calls with the same batch
        size must not overlap."""
        if batch > ONE_CTA_MAX_BATCH and batch not in self.ws:
            lib = _lib.load(require_device=True)
            nbytes = lib.mmssl_sampler_workspace_bytes(self.n_exist, batch)
            if nbytes < 0:
                raise _lib.MmsslLibraryError("mmssl_sampler_workspace_bytes failed")
            self.ws[batch] = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device=self.device)
        if self.exchange == "multicast" and batch not in self.ar:
            from .rowshard_step import MulticastAllReduce
            try:
                self.ar[batch] = MulticastAllReduce(3 * batch, self.device, self.group, ids=True)
                self.own[batch] = torch.zeros(3, batch, dtype=torch.int64, device=self.device)
            except RuntimeError:
                self.ar[batch] = None           # no NVSwitch multicast address: the NCCL all-reduce
        if self.exchange == "nccl":
            self.ar[batch] = None

    def sample_into(self, out: torch.Tensor, step_dev: torch.Tensor = None, step: int = 0) -> torch.Tensor:
        """Fills out[3, B] (int64: users, pos, neg; global ids) on every rank with the one-GPU sampler's batch.  A collective
        at world > 1.  `step_dev` (int32 device scalar) makes the launch replayable inside a CUDA graph."""
        lib = _lib.load(require_device=True)
        assert out.dtype == torch.int64 and out.dim() == 2 and out.shape[0] == 3 and out.is_contiguous()
        b = out.shape[1]
        self.reserve(b)
        ar = self.ar.get(b)
        part = self.own[b] if ar is not None else out
        args = (ptr(self.indptr), ptr(self.indices), ptr(self.exist), self.slot_lo, self.slot_hi, self.row0, self.n_exist, self.n_items,
                b, self.seed, ptr(step_dev), int(step))
        if b <= ONE_CTA_MAX_BATCH:
            _lib.check(lib.mmssl_sample_triples_owned(*args, ptr(self.claim), ptr(part[0]), ptr(part[1]), ptr(part[2]), stream()))
        else:
            ws = self.ws[b]
            _lib.check(lib.mmssl_sample_triples_multi_owned(*args, ptr(ws), ws.numel(), ptr(part[0]), ptr(part[1]), ptr(part[2]),
                                                            stream()))
        if ar is not None:
            ar.write_ids(part)
            ar.reduce_into(out)
        elif self.exchange is not None:         # every entry has one writer: the integer sum is exact
            dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.group)
        return out

    @classmethod
    def from_dataset(cls, sh, group=None, device="cuda", seed: int = 2022, exchange: str = "nccl") -> "ShardedTripleSampler":
        """From a ``dataset.ShardedDataset`` opened for this rank: its ``train_rows()`` and user partition."""
        return cls(sh.train_rows(), sh.part["user"], sh.rank, group=group, device=device, seed=seed, exchange=exchange)
