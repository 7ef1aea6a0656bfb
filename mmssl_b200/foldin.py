"""Fold-in: the top-k items for users the model never trained on -- or for trained users with interactions newer than the last
training run -- from their item lists, with the item side of the trained model held fixed.  No retraining.

By the closed form of the forward (SURVEY appendix A) a user's final row depends on the item side only through that user's own
row of the training graph A_ui: with r the user's distinct items and w = float32((|r| + 1e-8) ** -0.5) (csr_norm),
    u_{k+1} = w * sum_{j in r} i_k[j]  (k < K, row softmax on k = K-1),   Uv = w * sum Xv[j],   Ut = w * sum Xt[j]
    u_f = (u_0 + u_1 + ... + u_K) / (K + 1) + model_cat_rate * (normalize(Uv) + normalize(Ut))
where i_0 .. i_{K-1}, Xv, Xt are the eval-mode forward's item layer tables and projections (``Engine.forward(keep_fold=True)``)
and u_0 the user's id row after the id fusion.  ``mmssl_fold_users`` (csrc/rowops.cu) forms each sum as the training graph's SpMM
forms it, so a trained user's own training row folds to the forward's u_f row bit for bit (rows up to the SpMM's heavy cut of
1024 items; longer rows are summed in segment order where the forward uses float atomics, so they agree to fp32 rounding).

  ``FoldIn``         one GPU: ``fold(rows, users)`` -> [n, d] folded rows; ``topk(rows, k, users, exclude)`` -> (ids [n, k] int64,
                     scores [n, k] fp32); ``export(rows, k, out_dir, ...)`` writes ``{ids,scores,queries}.npy`` chunk by chunk.
  ``ShardedFoldIn``  a row-sharded model (rowshard_step.py): every rank gathers the K + 2 item-side tables and the final item table
                     once ((K + 3) * I * d * 4 bytes per rank) and folds the queries it is given; a query naming a trained user must go
                     to the rank that holds the user's row, new-user queries to any rank.  No id row crosses ranks.
  ``read(out_dir)``  (queries, ids, scores) of a fold-in export, either layout.

A query is an item list (``rows`` = an (indptr, indices) host int64 pair, ``dataset.held_csr`` builds one from a dict), sorted and
de-duplicated here (the training matrix is 0/1: an item counts once), plus optionally the id of a trained user (``users``, -1 for
a new user).  A trained user's u_0 is its row of the forward's u_0; a new user has u_0 = 0 -- and no row in the modality graphs, so
no id-fusion term -- while the layer mean still divides by K + 1, so scores are on the trained users' scale.  An empty row gives
what the forward gives a user without training items.  Ranking is recommend.py's: the query's own items are never listed;
exclude="train" also drops a trained user's training items, "seen" also its validation and test items (for new users both mean
the query row only).  Exports share recommend.py's file logic under the format ``mmssl_b200.foldin.v1``, ``queries.npy`` holding
each list's row number in the input; each of the four readers refuses the other formats."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import FoldTables, ptr, stream
from .parallel import RowPartition, all_gather_rows
from .recommend import (EXCLUDE, MANIFEST, Recommender, _Files, _manifests, _new_export_id, _rank_prefix, _read, _sharded_stale,
                        shared_export_id, union_csr)

FORMAT = "mmssl_b200.foldin.v1"
MAX_LAYERS = _lib.FOLD_MAX_LAYERS
_BAD_ITEM = "a query row holds an item id outside [0, n_items)"
_BAD_USER = "users holds an id that is neither -1 (a new user) nor a user of the model"

Rows = Tuple[np.ndarray, np.ndarray]


def row_weights(deg) -> np.ndarray:
    """The fp32 weight of a row of `deg` distinct items in the training graph: csr_norm's own expression on the fp32 row sums of a
    0/1 matrix (what ``Trainer`` and ``dataset.write_shards`` build A_ui with), so it is the graph's value bit for bit."""
    rs = np.asarray(deg).astype(np.float32)
    return np.asarray(np.power(rs + 1e-8, -0.5), np.float32)


def prepare_rows(rows, n_items: int) -> Rows:
    """(indptr, indices) host pair -> int64 CSR with every row sorted and de-duplicated; ids outside [0, n_items) are refused."""
    ip, ix = rows
    ip = np.asarray(ip, np.int64).reshape(-1)
    if ip.size < 1 or ip[0] != 0 or (np.diff(ip) < 0).any():
        raise ValueError("rows: indptr must start at 0 and not decrease")
    ix = np.asarray(ix, np.int64).reshape(-1)
    if ix.size < ip[-1]:
        raise ValueError(f"rows: indptr names {int(ip[-1])} entries, indices holds {ix.size}")
    ix = ix[:int(ip[-1])]
    if ix.size and (int(ix.min()) < 0 or int(ix.max()) >= n_items):
        raise ValueError(_BAD_ITEM)
    n = ip.size - 1
    r = np.repeat(np.arange(n, dtype=np.int64), np.diff(ip))
    key = np.unique(r * max(int(n_items), 1) + ix)
    rr, cc = key // max(int(n_items), 1), key % max(int(n_items), 1)
    out = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rr, minlength=n), out=out[1:])
    return out, cc


def take_rows(rows: Rows, users: np.ndarray) -> Rows:
    """The rows `users` of a host CSR, in that order (an empty row for -1)."""
    ip, ix = np.asarray(rows[0], np.int64), np.asarray(rows[1])
    ok = users >= 0
    u = np.where(ok, users, 0)
    lens = np.where(ok, ip[u + 1] - ip[u], 0)
    out = np.zeros(users.size + 1, np.int64)
    np.cumsum(lens, out=out[1:])
    starts = np.repeat(ip[u] - out[:-1], lens)
    return out, ix[starts + np.arange(int(out[-1]), dtype=np.int64)].astype(np.int64)


def _meta() -> dict:
    return dict(format=FORMAT, kind="foldin")


def _table(t: torch.Tensor, what: str, d: Optional[int] = None) -> torch.Tensor:
    t = t.detach()
    if t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2:
        raise TypeError(f"{what} must be a 2-D fp32 CUDA tensor")
    if d is not None and t.shape[1] != d:
        raise ValueError(f"{what} has width {t.shape[1]}, the other tables {d}")
    if t.stride(1) != 1 or t.stride(0) % 4 or t.data_ptr() % 16:
        t = t.contiguous().clone()
    return t


class FoldIn:
    """Folds item lists into user rows against fixed item-side tables, and ranks them against the final item table.
      u0:      [n_users, d] the forward's u_0 (id rows after the id fusion), or None (new users only);
      layers:  the K item layer tables i_0 .. i_{K-1} [n_items, d] (K <= MAX_LAYERS);
      xv, xt:  the eval-mode projections [n_items, d];  items: the final item table i_f [n_items, d];
      held:    optional (train, val, test) host CSRs over the users of u0 -- what exclude="train" / "seen" add for id queries.
    The tables are used as given (a snapshot of one forward): build a new FoldIn after the model changes."""

    def __init__(self, u0: Optional[torch.Tensor], layers: Sequence[torch.Tensor], xv: torch.Tensor, xt: torch.Tensor,
                 items: torch.Tensor, model_cat_rate: float = 0.55, held: Optional[Sequence[Rows]] = None):
        _lib.load(require_device=True)
        if len(layers) > MAX_LAYERS:
            raise ValueError(f"{len(layers)} GCN layers: the fold-in kernel is built for at most {MAX_LAYERS}")
        self.items = _table(items, "the final item table")
        self.n_items, self.d = self.items.shape
        if not _lib.load().mmssl_embed_width_supported(int(self.d)):
            raise ValueError(f"embedding width {self.d} is not supported")
        self.layers = tuple(_table(t, f"layer table {k}", self.d) for k, t in enumerate(layers))
        self.xv, self.xt = _table(xv, "Xv", self.d), _table(xt, "Xt", self.d)
        for t in self.layers + (self.xv, self.xt):
            if t.shape[0] != self.n_items:
                raise ValueError(f"an item-side table has {t.shape[0]} rows, the final item table {self.n_items}")
        self.u0 = None if u0 is None else _table(u0, "u0", self.d)
        self.n_users = 0 if u0 is None else self.u0.shape[0]
        self.K, self.rate = len(self.layers), float(model_cat_rate)
        self.held = None if held is None else tuple((np.asarray(a, np.int64), np.asarray(b)) for a, b in held)
        if self.held is not None and any(h[0].size != self.n_users + 1 for h in self.held):
            raise ValueError(f"the held rows must have one row per user ({self.n_users})")
        self.device = self.items.device
        self._desc = FoldTables()
        for k, t in enumerate(self.layers):
            self._desc.layer[k], self._desc.ld_layer[k] = t.data_ptr(), t.stride(0)
        self._desc.xv, self._desc.ldxv, self._desc.xt, self._desc.ldxt = \
            self.xv.data_ptr(), self.xv.stride(0), self.xt.data_ptr(), self.xt.stride(0)

    @classmethod
    def from_forward(cls, engine, P, feats, graphs, held: Optional[Sequence[Rows]] = None) -> "FoldIn":
        """From the eval-mode forward (no dropout) of a one-GPU model: ``Engine.forward(keep_fold=True)``."""
        outs, st = engine.forward(P, feats, graphs, None, want_sumsq=False, keep_fold=True)
        d = engine.d
        return cls(st.u0, st.i_layers, st.X2[:, :d], st.X2[:, d:], outs[1], engine.cat_rate, held)

    # -------------------------------------------------------------- queries
    def check_users(self, users, n: int) -> np.ndarray:
        if users is None:
            return np.full(n, -1, np.int64)
        ids = np.ascontiguousarray(np.asarray(users.cpu() if torch.is_tensor(users) else users, np.int64).reshape(-1))
        if ids.size != n:
            raise ValueError(f"users holds {ids.size} ids for {n} query rows")
        if ids.size and (int(ids.min()) < -1 or int(ids.max()) >= self.n_users):
            raise ValueError(_BAD_USER)
        return ids

    def _fold(self, q: Rows, users: np.ndarray) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(folded [n, d], indptr, indices on the device) of prepared rows."""
        n, dev = users.size, self.device
        ip, ix = torch.from_numpy(q[0]).to(dev), torch.from_numpy(q[1]).to(dev)
        out = torch.empty(n, self.d, dtype=torch.float32, device=dev)
        if n:
            w = torch.from_numpy(row_weights(np.diff(q[0]))).to(dev)
            us = torch.from_numpy(users).to(dev)
            u0 = self.u0
            _lib.check(_lib.load().mmssl_fold_users(ptr(ip), ptr(ix), ptr(us), ptr(w), n, ptr(u0), 0 if u0 is None else u0.stride(0),
                                                    self._desc, self.d, self.K, 1.0 / (self.K + 1), self.rate, ptr(out), out.stride(0),
                                                    stream()))
        return out, ip, ix

    def fold(self, rows, users=None) -> torch.Tensor:
        """[n, d] fp32 on the device: the final user row of each query (row i for query i)."""
        q = prepare_rows(rows, self.n_items)
        return self._fold(q, self.check_users(users, q[0].size - 1))[0]

    def _exclusion(self, q: Rows, users: np.ndarray, exclude: str) -> Optional[Rows]:
        """The rows a query's list skips beyond its own items (None: the query rows alone)."""
        if exclude not in EXCLUDE:
            raise ValueError(f"exclude must be one of {EXCLUDE}, not {exclude!r}")
        if self.held is None or not (users >= 0).any():
            return None
        held = self.held[:1] if exclude == "train" else self.held
        return union_csr(q, *(take_rows(h, users) for h in held))

    def _rank(self, q: Rows, users: np.ndarray, k: int, exclude: str):
        folded, ip, ix = self._fold(q, users)
        ex = self._exclusion(q, users, exclude)
        if ex is not None:
            ip, ix = torch.from_numpy(ex[0]).to(self.device), torch.from_numpy(ex[1]).to(self.device)
        if ix.numel() == 0:                          # every row empty: a valid pointer that no row reads
            ix = torch.zeros(1, dtype=torch.int64, device=self.device)
        return Recommender(self.items, (ip, ix), k).topk(folded, np.arange(users.size, dtype=np.int64))

    def topk(self, rows, k: int, users=None, exclude: str = "train") -> Tuple[torch.Tensor, torch.Tensor]:
        """(ids [n, k] int64, scores [n, k] fp32) on the device: the best k items of each folded query by recommend.py's order,
        its own items (and for an id query its training -- "seen": also validation and test -- items) never listed."""
        if int(k) < 1:
            raise ValueError("k must be >= 1")
        if exclude not in EXCLUDE:
            raise ValueError(f"exclude must be one of {EXCLUDE}, not {exclude!r}")
        q = prepare_rows(rows, self.n_items)
        return self._rank(q, self.check_users(users, q[0].size - 1), int(k), exclude)

    def _chunks(self, rows, k: int, users, exclude: str, chunk: int):
        """Yields (first row, ids [m, k] int32 host, scores [m, k] fp32 host) chunk by chunk of the prepared queries."""
        if chunk < 1:
            raise ValueError("chunk must be >= 1")
        q = prepare_rows(rows, self.n_items)
        n = q[0].size - 1
        us = self.check_users(users, n)
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            sub = (q[0][s:e + 1] - q[0][s], q[1][q[0][s]:q[0][e]])
            ids, sc = self._rank(sub, us[s:e], k, exclude)
            yield s, ids.to(torch.int32).cpu().numpy(), sc.cpu().numpy()

    def export(self, rows, k: int, out_dir: str, users=None, exclude: str = "train", chunk: int = 1 << 16,
               names: Optional[np.ndarray] = None, prefix: str = "", export_id: Optional[int] = None, stale=None) -> int:
        """Folds and ranks the queries ``chunk`` at a time into ``ids.npy`` (int32 [n, k]), ``scores.npy`` (fp32 [n, k]) and
        ``queries.npy`` (int64 [n]: each row's number in `rows`, or `names`) in out_dir, committed by ``manifest.json``
        (recommend.py's file logic).  Returns n."""
        if int(k) < 1:
            raise ValueError("k must be >= 1")
        if exclude not in EXCLUDE:
            raise ValueError(f"exclude must be one of {EXCLUDE}, not {exclude!r}")
        n = np.asarray(rows[0]).size - 1
        if stale is None:
            _, ranks = _manifests(out_dir)
            stale = [MANIFEST] + list(ranks.values())
        files = _Files(out_dir, prefix, n, int(k), _new_export_id() if export_id is None else export_id, stale, "queries", _meta())
        try:
            if n:
                files.arr["queries"][:] = np.arange(n, dtype=np.int64) if names is None else names
            for s, ids, sc in self._chunks(rows, int(k), users, exclude, chunk):
                files.arr["ids"][s:s + ids.shape[0]] = ids
                files.arr["scores"][s:s + ids.shape[0]] = sc
            files.commit()
        except BaseException:
            files.discard()
            raise
        return n


def read(out_dir: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(queries [n] int64, ids [n, k] int32, scores [n, k] fp32) of the committed fold-in export in out_dir, either layout
    (recommend.read's rules); a recommendation, similar-items or audience export is refused."""
    return _read(out_dir, "queries", FORMAT, "fold-in")


class ShardedFoldIn:
    """``FoldIn`` of a model whose tables are row-sharded over the ranks of a process group (rowshard_step.py): one per rank.  The
    item-side tables and the final item table are gathered once, at construction ((K + 3) * n_items * d * 4 bytes per rank); the
    rank keeps its own block of u_0 and of the held rows.  ``topk`` / ``fold`` / ``export`` take the queries this rank is given:
    a query naming a trained user must be given to the rank that holds that user's row (``mine``), new-user queries (-1) may go
    to any rank; other user ids are refused.  A folded row depends only on its row, its u_0 row and the item-side tables, so every
    list is bitwise the one-GPU ``FoldIn``'s on the gathered tables."""

    def __init__(self, local: FoldIn, part_u: RowPartition, rank: int):
        self.local, self.pu, self.rank_id = local, part_u, int(rank)
        self.lo, self.hi = part_u.bounds(self.rank_id)
        self.n_users, self.n_items, self.d, self.device = part_u.n, local.n_items, local.d, local.device

    @classmethod
    def from_shards(cls, tables, part_u: RowPartition, part_i: RowPartition, rank: int, model_cat_rate: float = 0.55,
                    held: Optional[Sequence[Rows]] = None, group=None) -> "ShardedFoldIn":
        """Collective.  tables: ``RowShardedHotStep.fold_tables()`` of this rank; held: optional (train, val, test) CSRs of the
        rank's user block with local row numbers (``dataset.ShardedDataset``: train_rows(), held("val"), held("test"))."""
        g = lambda t: all_gather_rows(t.detach().contiguous(), part_i, group)
        layers = [g(t) for t in tables["layers"]]
        local = FoldIn(tables["u0"], layers, g(tables["xv"]), g(tables["xt"]), g(tables["i_f"]), model_cat_rate, held)
        return cls(local, part_u, rank)

    @classmethod
    def from_dataset(cls, tables, sh, model_cat_rate: float = 0.55, group=None) -> "ShardedFoldIn":
        """Collective.  ``from_shards`` with the held rows of a ``dataset.ShardedDataset`` (rank and world as it was opened with)."""
        pair = lambda b: (np.asarray(b.indptr, np.int64), np.asarray(b.indices, np.int64))
        held = (pair(sh.train_rows()), pair(sh.held("val")), pair(sh.held("test")))
        return cls.from_shards(tables, sh.part["user"], sh.part["item"], sh.rank, model_cat_rate, held, group)

    def mine(self, users: np.ndarray) -> np.ndarray:
        """Positions in `users` of the id queries this rank holds the user of."""
        return np.nonzero((users >= self.lo) & (users < self.hi))[0]

    def _local_users(self, users, n: int) -> np.ndarray:
        if users is None:
            return np.full(n, -1, np.int64)
        ids = np.ascontiguousarray(np.asarray(users.cpu() if torch.is_tensor(users) else users, np.int64).reshape(-1))
        if ids.size != n:
            raise ValueError(f"users holds {ids.size} ids for {n} query rows")
        bad = (ids != -1) & ((ids < self.lo) | (ids >= self.hi))
        if bad.any():
            u = int(ids[np.nonzero(bad)[0][0]])
            raise ValueError(f"user {u} is not held by rank {self.rank_id} (users [{self.lo}, {self.hi})): give an id query to "
                             "the rank that holds the user, or -1 for a new user")
        return np.where(ids >= 0, ids - self.lo, -1)

    def fold(self, rows, users=None) -> torch.Tensor:
        n = np.asarray(rows[0]).size - 1
        return self.local.fold(rows, self._local_users(users, n))

    def topk(self, rows, k: int, users=None, exclude: str = "train"):
        n = np.asarray(rows[0]).size - 1
        return self.local.topk(rows, k, self._local_users(users, n), exclude)

    def export(self, rows, k: int, out_dir: str, users=None, exclude: str = "train", chunk: int = 1 << 16,
               names: Optional[np.ndarray] = None, group=None) -> int:
        """Collective (the shared export id).  Writes ``rankRRRRR-of-WWWWW.{ids,scores,queries}.npy`` with this rank's queries, in
        their given order (``queries.npy``: `names`, e.g. their row numbers in a file every rank read, default 0..n-1) and commits
        them with ``rankRRRRR-of-WWWWW.json``.  Returns the number of rows written."""
        n = np.asarray(rows[0]).size - 1
        us = self._local_users(users, n)
        world = self.pu.world
        export_id = shared_export_id(self.rank_id, world, self.device, group)
        return self.local.export(rows, k, out_dir, us, exclude, chunk, names, _rank_prefix(self.rank_id, world), export_id,
                                 _sharded_stale(out_dir, self.rank_id, world))
