"""Device-side triple sampler (SURVEY 8f "next" #1): the reference's ``Data.sample``
(utility/load_data.py:153-191) as CUDA kernels, so a training step needs no host input at all.
Batches of up to 1024 triples take one single-CTA launch; larger batches take an exact multi-CTA
radix select over all users that have a training item (csrc/sampler.cu)."""
from __future__ import annotations

import numpy as np
import torch

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
