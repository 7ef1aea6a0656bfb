"""Evaluation on the device (SURVEY 8f "next" #3): host-side mirror of the reference's
``utility/batch_test.py:test_torch`` (same arguments, same result dict) over ``mmssl_eval_rank`` /
``mmssl_eval_reduce``.  The reference scores 2048 users at a time, copies the dense score rows to the host and
ranks them in a ``multiprocessing.Pool`` with ``heapq`` (batch_test.py:112-169); here ranking, masking of the
training items, hit marking and the metrics are one kernel and only the [4, len(Ks)] result leaves the GPU.
``test_flag='full'`` (batch_test.py:38-68, 104-107) adds the per-user ROC-AUC over all non-training items
(``mmssl_eval_rank_full``): the same sweep, no host sort.  Ks is any list of cut-offs >= 1 (parser.py:63), unsorted or with
duplicates: up to 8 cut-offs of at most 64 go to the shared-memory kernel, any other list to ``mmssl_eval_rank_wide``.
``ShardedEvaluator`` is the same evaluation for a row-sharded model (rowshard_step.py), on the ranks that hold it, with the
one-GPU result bit for bit."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Sequence

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from ._lib import ptr, stream
from .parallel import RowPartition, all_gather_rows

_BAD_USER = "users_to_test holds an id outside [0, n_users): the ranking kernel indexes the CSR row pointers with it"


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
        self._setup(n_users, n_items, Ks, device, test_flag)
        self._set_rows(_rows_to_csr(train_items, n_users, self.device), _rows_to_csr(test_set, n_users, self.device),
                       _rows_to_csr(val_set, n_users, self.device))

    @classmethod
    def _from_csr(cls, train, test, val, n_users: int, n_items: int, Ks: Sequence[int], device, test_flag: str) -> "Evaluator":
        """The same evaluator over rows that are already (indptr, indices) int64 tensors on `device`, sorted within each row
        (ShardedEvaluator: a rank's user block, built from the shard arrays without per-user dicts)."""
        ev = cls.__new__(cls)
        ev._setup(n_users, n_items, Ks, device, test_flag)
        ev._set_rows(train, test, val)
        return ev

    def _setup(self, n_users, n_items, Ks, device, test_flag) -> None:
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

    def _set_rows(self, train, test, val) -> None:
        self.train = train
        self.held = {False: test, True: val}
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
            raise ValueError(_BAD_USER)
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
        return _test_result(self.rank(ua_embeddings, ia_embeddings, users_to_test, is_val), self.test_flag, self.device)


def _test_result(out: Dict[str, torch.Tensor], test_flag: str, device) -> Dict[str, object]:
    """batch_test.py's result dict from rank()'s output: the [4, nK] metrics and, in full mode, the mean of the per-user AUC."""
    res = out["result"].cpu().numpy()
    auc = 0.
    if test_flag == "full":
        mean = torch.zeros(1, dtype=torch.float64, device=device)
        _lib.check(_lib.load().mmssl_eval_reduce(ptr(out["auc"]), out["auc"].numel(), 1, ptr(mean), stream()))
        auc = float(mean.cpu()[0])
    return {"precision": res[0].copy(), "recall": res[1].copy(), "ndcg": res[2].copy(), "hit_ratio": res[3].copy(), "auc": auc}


def _device_csr(indptr, indices, device) -> tuple:
    """(indptr, indices) host arrays (indices int32 or int64, e.g. views of the shard maps) -> the kernels' int64 tensors; the
    indices travel as they are and are widened on the device."""
    ip = torch.from_numpy(np.array(indptr, dtype=np.int64)).to(device)
    ix = torch.from_numpy(np.array(indices, dtype=np.int32 if np.asarray(indices).dtype.itemsize == 4 else np.int64)).to(device)
    return ip, ix.to(torch.int64)


def _block_rows(rows: Mapping[int, Sequence[int]], part: RowPartition, rank: int) -> tuple:
    """dict user -> item list -> CSR of the rank's user block (local row ids, sorted rows, padding rows empty)."""
    from .dataset import held_csr
    lo, hi = part.bounds(rank)
    return held_csr({int(u) - lo: its for u, its in rows.items() if lo <= int(u) < hi}, part.block)


class ShardedEvaluator:
    """``Evaluator`` for a model whose tables are row-sharded over the ranks of a process group (rowshard_step.py): one per
    rank, holding only the train / test / val rows of the rank's user block.

    ``rank(u_local, i_local, users_to_test, is_val)`` takes the rank's padded [block, d] rows of the final user and item tables
    and the same list of global user ids on every rank, and
      1. all-gathers the item table (n_items x d fp32 on every rank: 1 GB at 1M items, d = 256);
      2. ranks the listed users that fall in the rank's block, with local ids against the rank's rows, by the same kernels
         (``Evaluator.rank``'s launch code; item ids stay global, so the tie rule -- equal score, lower id first -- is the same);
      3. all-gathers the per-user metric rows (and per-user AUC in full mode), padded to the largest per-rank count, places them
         at their positions in ``users_to_test`` and runs ``mmssl_eval_reduce`` over the assembled [n, 4, nK] buffer.
    A per-user row depends only on that user's vector, the item table and the user's rows, and the reduction runs over the rows
    in list order as on one GPU, so every rank's result (and mean AUC) is bitwise what ``Evaluator`` returns on the gathered
    tables.  The gathered and the assembled rows take n * (4 nK + 1) * 8 bytes each: about 1 GB at 10M users and three
    cut-offs.  The ranked lists are not gathered: each rank returns its own, with their positions in ``users_to_test``."""

    _local_cls = Evaluator       # the class itself, bound when this module is imported

    def __init__(self, train, test, val, part_u: RowPartition, part_i: RowPartition, rank: int, n_items: int,
                 Ks: Sequence[int] = (10, 20, 50), test_flag: str = "part", group=None, device="cuda"):
        """train / test / val: (indptr, indices) of the rank's user block -- indptr [block + 1] rebased to 0, indices global
        item ids sorted within each row (int32 or int64)."""
        if int(n_items) != part_i.n:
            raise ValueError(f"n_items {n_items} does not match the item partition ({part_i.n} rows)")
        for name, (ip, _) in (("train", train), ("test", test), ("val", val)):
            if len(ip) != part_u.block + 1:
                raise ValueError(f"{name} rows: indptr of {len(ip)} entries, the user block needs {part_u.block + 1}")
        self.pu, self.pi, self.rank_id, self.group = part_u, part_i, int(rank), group
        self.n_users, self.n_items = part_u.n, int(n_items)
        dev = torch.device(device)
        rows = [_device_csr(ip, ix, dev) for ip, ix in (train, test, val)]
        self._local = self._local_cls._from_csr(*rows, part_u.block, n_items, Ks, dev, test_flag)
        self.Ks, self.test_flag, self.wide, self.device = self._local.Ks, test_flag, self._local.wide, dev

    @classmethod
    def from_shards(cls, sh, Ks: Sequence[int] = (10, 20, 50), test_flag: str = "part", group=None, device="cuda") -> "ShardedEvaluator":
        """From ``dataset.ShardedDataset`` (rank and world as it was opened with): training rows = the pattern of the rank's ``ui``
        rows, held-out rows from the ``val`` / ``test`` arrays."""
        pair = lambda b: (b.indptr, b.indices)
        return cls(pair(sh.train_rows()), pair(sh.held("test")), pair(sh.held("val")), sh.part["user"], sh.part["item"], sh.rank,
                   sh.n_items, Ks, test_flag, group, device)

    @classmethod
    def from_rows(cls, train_items, test_set, val_set, n_users: int, n_items: int, part_u: RowPartition, part_i: RowPartition,
                  rank: int, Ks: Sequence[int] = (10, 20, 50), test_flag: str = "part", group=None, device="cuda") -> "ShardedEvaluator":
        """From the reference's dicts (``Data.train_items`` / ``test_set`` / ``val_set``); every rank keeps its block's rows."""
        if part_u.n != int(n_users):
            raise ValueError(f"n_users {n_users} does not match the user partition ({part_u.n} rows)")
        rows = [_block_rows(r, part_u, rank) for r in (train_items, test_set, val_set)]
        return cls(*rows, part_u, part_i, rank, n_items, Ks, test_flag, group, device)

    # ------------------------------------------------------------------ the phases of rank()
    def check_users(self, users_to_test) -> np.ndarray:
        ids = users_to_test.detach().cpu().numpy() if torch.is_tensor(users_to_test) else list(users_to_test)
        ids = np.asarray(ids, np.int64).reshape(-1)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= self.n_users):
            raise ValueError(_BAD_USER)
        return ids

    def gather_items(self, i_local: torch.Tensor) -> torch.Tensor:
        """[block, d] item rows of every rank -> the full [n_items, d] table."""
        return all_gather_rows(i_local.detach(), self.pi, self.group)

    def rank_local(self, u_local: torch.Tensor, items: torch.Tensor, ids: np.ndarray, is_val: bool):
        """Ranks the entries of `ids` in the rank's user block.  Returns (Evaluator.rank's output, their positions in `ids`)."""
        lo = self.rank_id * self.pu.block
        mine = np.nonzero(ids // self.pu.block == self.rank_id)[0]
        if mine.size == 0:           # none of the listed users is here: no launch (the kernels take no empty outputs)
            kmax, nk, dev = max(self.Ks), len(self.Ks), self.device
            out = dict(ranked=torch.empty(0, kmax, dtype=torch.int32, device=dev),
                       ranked_scores=torch.empty(0, kmax, dtype=torch.float32, device=dev),
                       hits=torch.empty(0, kmax, dtype=torch.int32, device=dev),
                       per_user=torch.empty(0, 4, nk, dtype=torch.float64, device=dev))
            if self.test_flag == "full":
                out["auc"] = torch.empty(0, dtype=torch.float64, device=dev)
            return out, mine
        return self._local.rank(u_local, items, ids[mine] - lo, is_val), mine

    def combine(self, local: Dict[str, torch.Tensor], ids: np.ndarray) -> Dict[str, torch.Tensor]:
        """Every rank's per-user rows at their positions in `ids`, and the result reduced over them in that order."""
        nk, n, world, dev = len(self.Ks), ids.size, self.pu.world, self.device
        full = self.test_flag == "full"
        w = 4 * nk + (1 if full else 0)
        owner = ids // self.pu.block
        counts = np.bincount(owner, minlength=world)
        m = int(counts.max()) if n else 0
        rows = torch.empty(n, w, dtype=torch.float64, device=dev)
        if n:
            k = int(counts[self.rank_id])
            part = torch.zeros(m, w, dtype=torch.float64, device=dev)
            part[:k, :4 * nk] = local["per_user"].reshape(k, 4 * nk)
            if full:
                part[:k, 4 * nk] = local["auc"]
            if world > 1:
                every = torch.empty(world * m, w, dtype=torch.float64, device=dev)
                dist.all_gather_into_tensor(every, part, group=self.group)
            else:
                every = part
            # owners in list order, grouped by rank: the r-th group is rank r's rows 0 .. counts[r] - 1
            dst = np.argsort(owner, kind="stable")
            src = np.concatenate([r * m + np.arange(counts[r], dtype=np.int64) for r in range(world)])
            rows[torch.from_numpy(dst).to(dev)] = every[torch.from_numpy(src).to(dev)]
        per_user = rows[:, :4 * nk].contiguous().view(n, 4, nk)
        result = torch.zeros(4, nk, dtype=torch.float64, device=dev)
        _lib.check(_lib.load().mmssl_eval_reduce(ptr(per_user), n, 4 * nk, ptr(result), stream()))
        out = dict(per_user=per_user, result=result)
        if full:
            out["auc"] = rows[:, 4 * nk].contiguous()
        return out

    def rank(self, u_local: torch.Tensor, i_local: torch.Tensor, users_to_test, is_val: bool) -> Dict[str, torch.Tensor]:
        """Collective.  Device tensors: result [4, nK] and per_user [n, 4, nK] fp64 in list order, in full mode auc [n] fp64; the
        rank's own ranked / ranked_scores / hits rows and ``positions`` (host int64) -- where they stand in users_to_test."""
        ids = self.check_users(users_to_test)
        items = self.gather_items(i_local)
        local, mine = self.rank_local(u_local, items, ids, is_val)
        out = self.combine(local, ids)
        out.update(ranked=local["ranked"], ranked_scores=local["ranked_scores"], hits=local["hits"], positions=torch.from_numpy(mine))
        return out

    def test_torch(self, u_local, i_local, users_to_test, is_val, drop_flag=False, batch_test_flag=False):
        """Collective.  ``Evaluator.test_torch``'s result dict, identical on every rank."""
        return _test_result(self.rank(u_local, i_local, users_to_test, is_val), self.test_flag, self.device)
