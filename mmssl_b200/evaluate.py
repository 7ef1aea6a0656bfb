"""Evaluation on the device (SURVEY 8f "next" #3): host-side mirror of the reference's
``utility/batch_test.py:test_torch`` (same arguments, same result dict) over ``mmssl_eval_rank`` /
``mmssl_eval_reduce``.  The reference scores 2048 users at a time, copies the dense score rows to the host and
ranks them in a ``multiprocessing.Pool`` with ``heapq`` (batch_test.py:112-169); here ranking, masking of the
training items, hit marking and the metrics are one kernel and only the [4, len(Ks)] result leaves the GPU.
``test_flag='full'`` (batch_test.py:38-68, 104-107) adds the per-user ROC-AUC over all non-training items
(``mmssl_eval_rank_full``): the same sweep, no host sort.  Ks is any list of cut-offs >= 1 (parser.py:63), unsorted or with
duplicates: up to 8 cut-offs of at most 64 go to the shared-memory kernel, any other list to ``mmssl_eval_rank_wide``."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import ptr, stream


def _rows_to_csr(rows: Mapping[int, Sequence[int]], n_users: int, device) -> tuple:
    """dict user -> item list (Data.train_items / test_set / val_set, load_data.py:62-88) -> CSR with sorted rows."""
    indptr = np.zeros(n_users + 1, np.int64)
    for u, its in rows.items():
        indptr[int(u) + 1] = len(its)
    np.cumsum(indptr, out=indptr)
    indices = np.empty(int(indptr[-1]), np.int64)
    for u, its in rows.items():
        b = indptr[int(u)]
        indices[b:b + len(its)] = np.sort(np.asarray(its, np.int64))
    return torch.from_numpy(indptr).to(device), torch.from_numpy(indices).to(device)


class Evaluator:
    """``Evaluator(data_generator.train_items, data_generator.test_set, data_generator.val_set, n_users, n_items, Ks)``
    then ``test_torch(ua_embeddings, ia_embeddings, users_to_test, is_val)`` exactly like batch_test.py:112.
    ``test_flag`` is the reference's ``--test_flag`` (parser.py:16): 'part' (auc 0.) or 'full' (mean per-user ROC-AUC)."""

    def __init__(self, train_items: Mapping[int, Sequence[int]], test_set: Mapping[int, Sequence[int]],
                 val_set: Mapping[int, Sequence[int]], n_users: int, n_items: int, Ks: Sequence[int] = (10, 20, 50), device="cuda",
                 test_flag: str = "part"):
        if test_flag not in ("part", "full"):
            raise ValueError(f"test_flag must be 'part' or 'full', not {test_flag!r}")
        self.test_flag = test_flag
        _lib.load(require_device=True)
        self.n_users, self.n_items = int(n_users), int(n_items)
        self.Ks = [int(k) for k in Ks]
        if not self.Ks or min(self.Ks) < 1:
            raise ValueError("Ks: at least one cut-off, each >= 1")
        # the kernel with 512-key shared buffers and a 64-bit hit mask takes up to 8 cut-offs of at most 64
        self.wide = len(self.Ks) > 8 or max(self.Ks) > 64
        self.device = torch.device(device)
        self.train = _rows_to_csr(train_items, n_users, self.device)
        self.held = {False: _rows_to_csr(test_set, n_users, self.device), True: _rows_to_csr(val_set, n_users, self.device)}
        self._held_len = {k: np.diff(v[0].cpu().numpy()) for k, v in self.held.items()}
        self._ks = (C.c_int32 * len(self.Ks))(*self.Ks)
        self._ks_dev = torch.tensor(self.Ks, dtype=torch.int32).to(self.device) if self.wide else None

    def rank(self, ua_embeddings: torch.Tensor, ia_embeddings: torch.Tensor, users_to_test, is_val: bool,
             want_scores: bool = False) -> Dict[str, torch.Tensor]:
        """Device tensors: ranked [n, kmax] int32, ranked_scores, hits, per_user [n, 4, nK] fp64, result [4, nK] fp64;
        in full mode also auc [n] fp64 (NaN for a user with one class only, like sklearn)."""
        lib = _lib.load(require_device=True)
        ua = ua_embeddings.detach()
        ia = ia_embeddings.detach()
        if ua.dtype != torch.float32 or ia.dtype != torch.float32 or not ua.is_cuda or not ia.is_cuda:
            raise TypeError("embeddings must be fp32 CUDA tensors")
        if ua.stride(1) != 1 or ia.stride(1) != 1:
            ua, ia = ua.contiguous(), ia.contiguous()
        if ia.stride(0) % 4 or ia.data_ptr() % 16:
            ia = ia.contiguous().clone()
        if ia.shape[0] != self.n_items or ua.shape[1] != ia.shape[1]:
            raise ValueError("embedding tables do not match the evaluator's shapes")
        ids = torch.as_tensor(list(users_to_test) if not torch.is_tensor(users_to_test) else users_to_test)
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= min(self.n_users, ua.shape[0])):
            raise ValueError("users_to_test holds an id outside [0, n_users): the ranking kernel indexes the CSR row pointers with it")
        users_np = np.asarray(list(users_to_test), np.int64)
        users = torch.as_tensor(users_np).to(self.device)
        n, kmax, nk, d = users.numel(), max(self.Ks), len(self.Ks), ua.shape[1]
        dev = self.device
        ranked = torch.empty(n, kmax, dtype=torch.int32, device=dev)
        rscore = torch.empty(n, kmax, dtype=torch.float32, device=dev)
        hits = torch.empty(n, kmax, dtype=torch.int32, device=dev)
        per_user = torch.empty(n, 4, nk, dtype=torch.float64, device=dev)
        result = torch.zeros(4, nk, dtype=torch.float64, device=dev)
        scores = torch.empty(n, self.n_items, dtype=torch.float32, device=dev) if want_scores else None
        held = self.held[bool(is_val)]
        head = (ptr(ua), ua.stride(0), ptr(ia), ia.stride(0), self.n_items, d, ptr(users), n, ptr(self.train[0]), ptr(self.train[1]),
                ptr(held[0]), ptr(held[1]), self._ks)
        ks = (ptr(self._ks_dev), nk) if self.wide else (nk,)
        args = head + ks + (ptr(ranked), ptr(rscore), ptr(hits), ptr(per_user), ptr(scores))
        out = dict(ranked=ranked, ranked_scores=rscore, hits=hits, per_user=per_user, result=result)
        auc = ws = off = None
        if self.test_flag == "full":
            # users whose held-out row does not fit the kernel's shared-memory stage sort their positives in a
            # workspace slot of next_pow2(row length) keys
            lens = self._held_len[bool(is_val)][users_np]
            slot = np.zeros(n, np.int64)
            for k in np.nonzero(lens > lib.mmssl_eval_full_stage())[0]:
                slot[k] = 1 << int(lens[k] - 1).bit_length()
            off = torch.from_numpy(np.cumsum(slot) - slot).to(dev)
            ws = torch.empty(int(slot.sum()), dtype=torch.int32, device=dev) if slot.sum() else None
            auc = torch.empty(n, dtype=torch.float64, device=dev)
            out["auc"] = auc
        if self.wide:
            nbytes = lib.mmssl_eval_wide_workspace_bytes(n, kmax, self.n_items, d)
            key_ws = torch.empty(nbytes // 8, dtype=torch.int64, device=dev) if nbytes else None
            _lib.check(lib.mmssl_eval_rank_wide(*args, ptr(auc), ptr(ws), ptr(off), ptr(key_ws), stream()))
        elif self.test_flag == "full":
            _lib.check(lib.mmssl_eval_rank_full(*args, ptr(auc), ptr(ws), ptr(off), stream()))
        else:
            _lib.check(lib.mmssl_eval_rank(*args, stream()))
        _lib.check(lib.mmssl_eval_reduce(ptr(per_user), n, 4 * nk, ptr(result), stream()))
        if want_scores:
            out["scores"] = scores
        return out

    def test_torch(self, ua_embeddings, ia_embeddings, users_to_test, is_val, drop_flag=False, batch_test_flag=False):
        """Same signature and result as batch_test.py:112-169 ('auc' is 0. in the default test_flag == 'part' mode, the mean
        per-user ROC-AUC in 'full' mode -- NaN as soon as one evaluated user has a single class, like the reference)."""
        out = self.rank(ua_embeddings, ia_embeddings, users_to_test, is_val)
        res = out["result"].cpu().numpy()
        auc = 0.
        if self.test_flag == "full":
            mean = torch.zeros(1, dtype=torch.float64, device=self.device)
            _lib.check(_lib.load().mmssl_eval_reduce(ptr(out["auc"]), out["auc"].numel(), 1, ptr(mean), stream()))
            auc = float(mean.cpu()[0])
        return {"precision": res[0].copy(), "recall": res[1].copy(), "ndcg": res[2].copy(), "hit_ratio": res[3].copy(), "auc": auc}
