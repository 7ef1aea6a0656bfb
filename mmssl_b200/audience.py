"""Audiences: the top-k users of each listed item -- which users should see it (targeting, push campaigns, a new item's launch) --
on the device, with no [items x users] score matrix anywhere.

  ``Audience(user_table, exclude, k)``   one GPU: ``topk(item_table, items)`` -> (ids [n, k] int64 user ids, scores [n, k] fp32) on
                                         the device; ``export(item_table, items, out_dir)`` ranks the items chunk by chunk into
                                         ``ids.npy`` / ``scores.npy`` / ``items.npy``.
  ``ShardedAudience``                    a row-sharded model (rowshard_step.py) on the ranks that hold it: every rank gathers the
                                         item table once, ranks the listed items against its own user rows and sends each partial
                                         list to the rank that owns the item, which merges them; the user table is never gathered.
                                         ``export`` writes ``rankRRRRR-of-WWWWW.{ids,scores,items}.npy`` per rank.
  ``read(out_dir)``                      (items, ids, scores) of either layout.

Ranking is recommend.py's with the roles of the tables swapped: the items are the queries, the users the candidates, and the
exclusion CSR has one row per item listing the users who must not get it (``transpose_csr`` of recommend.exclusion_rows):
"train" -- the users who had the item in training, so the score of a pair in an audience list is, bit for bit, its score in that
user's ``Recommender`` list -- or "seen", which also drops the users holding it in val or test.  Best score first, equal scores
lower user id first, -1 (score 0) past the end of a list shorter than k.  A call with few items is ranked over slices of the users
and merged (``Recommender._slices``), with the same lists.  Exports share recommend.py's file logic; the manifest's format is
``mmssl_b200.audience.v1`` and each of recommend.read / similar.read / audience.read refuses the others' directories."""
from __future__ import annotations

from typing import Mapping, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from .dataset import held_csr
from .evaluate import _block_rows, _device_csr
from .parallel import RowPartition, all_gather_rows
from .recommend import (EXCLUDE, MANIFEST, Recommender, _Files, _host_ids, _manifests, _new_export_id, _rank_prefix, _read,
                        _sharded_stale, exclusion_rows, merge_lists, shared_export_id, union_csr)

FORMAT = "mmssl_b200.audience.v1"
_BAD_ITEM = "items holds an id outside [0, n_items)"


def transpose_csr(indptr, indices, n_cols: int) -> Tuple[np.ndarray, np.ndarray]:
    """CSR of rows -> CSR of its n_cols columns (host arrays): row c of the result lists, ascending, the rows whose entries hold
    c.  Turns the user -> items exclusion rows into the item -> users rows an audience excludes.  Entries outside [0, n_cols)
    are dropped: no item query reaches them (the reference's held-out rows may name ids past the training items, which the
    recommendation sweep likewise never meets)."""
    ip = np.asarray(indptr, np.int64)
    ix = np.asarray(indices)[int(ip[0]):int(ip[-1])].astype(np.int64)
    rows = np.repeat(np.arange(ip.size - 1, dtype=np.int64), np.diff(ip))
    keep = (ix >= 0) & (ix < n_cols)
    ix, rows = ix[keep], rows[keep]
    order = np.argsort(ix, kind="stable")               # rows stay ascending within each column
    out = np.zeros(n_cols + 1, np.int64)
    np.cumsum(np.bincount(ix, minlength=n_cols), out=out[1:])
    return out, rows[order]


def _meta() -> dict:
    return dict(format=FORMAT, kind="audience")


class Audience:
    """Top-k users of items against one user table.  ``exclude`` is (indptr [n_items + 1], indices) int64 on the table's device:
    per item the user ids it must not be shown to, sorted within each row (``from_rows`` builds it from the reference's dicts);
    its row count is the item count.  A ``Recommender`` with the tables' roles swapped does the ranking."""

    def __init__(self, user_table: torch.Tensor, exclude: Tuple[torch.Tensor, torch.Tensor], k: int):
        self.rec = Recommender(user_table, exclude, k)
        self.k, self.n_users, self.n_items, self.device = self.rec.k, self.rec.n_items, self.rec.n_users, self.rec.device

    @classmethod
    def from_rows(cls, user_table: torch.Tensor, train_items: Mapping[int, Sequence[int]], test_set, val_set, n_items: int, k: int,
                  exclude: str = "train") -> "Audience":
        """From the reference's dicts (``Data.train_items`` / ``test_set`` / ``val_set``) and an exclusion set name."""
        rows = held_csr(exclusion_rows(train_items, test_set, val_set, exclude), user_table.shape[0])
        return cls(user_table, _device_csr(*transpose_csr(*rows, int(n_items)), user_table.device), k)

    def check_items(self, items, n_rows: int) -> np.ndarray:
        ids = _host_ids(items)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= min(self.n_items, n_rows)):
            raise ValueError(_BAD_ITEM)
        return ids

    def topk(self, item_table: torch.Tensor, items) -> Tuple[torch.Tensor, torch.Tensor]:
        """(ids [n, k] int64 user ids, scores [n, k] fp32) on the device, row i for items[i]; n == 0 launches nothing."""
        ia = self.rec._user_table(item_table)
        return self.rec.topk(ia, self.check_items(items, ia.shape[0]))

    def export(self, item_table: torch.Tensor, items, out_dir: str, chunk: int = 1 << 16) -> int:
        """Ranks `items` ``chunk`` at a time into ``ids.npy`` (int32 [n, k] user ids), ``scores.npy`` (fp32 [n, k]) and ``items.npy``
        (int64 [n]) in out_dir and commits them with ``manifest.json`` (recommend.Recommender.export's file logic).  Returns n."""
        ia = self.rec._user_table(item_table)
        ids = self.check_items(items, ia.shape[0])
        _, ranks = _manifests(out_dir)
        return self.rec._export(ia, ids, ids, out_dir, chunk, "", _new_export_id(), [MANIFEST] + list(ranks.values()), "items",
                                _meta())


def read(out_dir: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(items [n] int64, ids [n, k] int32 user ids, scores [n, k] fp32) of the committed audience export in out_dir, either layout
    (recommend.read's rules: rank files in ascending item order, an incomplete row-sharded export refused); a recommendation or
    similar-items export is refused."""
    return _read(out_dir, "items", FORMAT, "audience")


class ShardedAudience:
    """``Audience`` of a model whose tables are row-sharded over the ranks of a process group (rowshard_step.py): one per rank,
    holding the exclusion rows of its own user block ([n_items + 1] rows of local user ids).  ``topk`` / ``export`` take the rank's
    padded [block, d] rows of the final user and item tables (``RowShardedHotStep.final_embeddings``) and the same list of global
    item ids on every rank.  Every rank gathers the item table once, then, chunk by chunk of the listed items, collectively:
      1. ranks every item of the chunk against its real user rows (padding rows are never candidates) into a partial list, with
         its block's base added to the user ids;
      2. sends each partial list to the rank that owns the item (``exchange``: one all-to-all);
      3. merges the world's partial lists of the items it owns (``mmssl_topk_merge``).
    The user table never travels.  A partial list holds the best k of the rank's users by the one-GPU keys, so the merged list is
    bitwise the one-GPU ``Audience``'s on the gathered tables; each rank returns and writes the lists of its own items."""

    def __init__(self, exclude, part_u: RowPartition, part_i: RowPartition, rank: int, k: int, group=None, device="cuda"):
        """exclude: (indptr [n_items + 1], indices: local user ids of the rank's block, sorted within each row)."""
        if len(exclude[0]) != part_i.n + 1:
            raise ValueError(f"exclusion rows: indptr of {len(exclude[0])} entries, the items need {part_i.n + 1}")
        self.pu, self.pi, self.rank_id, self.group = part_u, part_i, int(rank), group
        self.n_users, self.n_items, self.k = part_u.n, part_i.n, int(k)
        if self.k < 1:
            raise ValueError("k must be >= 1")
        lo, hi = part_u.bounds(self.rank_id)
        self.base, self.n_real = lo, hi - lo
        self.device = torch.device(device)
        self.exclude = _device_csr(exclude[0], exclude[1], self.device)

    @classmethod
    def from_shards(cls, sh, k: int, exclude: str = "train", group=None, device="cuda") -> "ShardedAudience":
        """From ``dataset.ShardedDataset`` (rank and world as it was opened with): "train" = the rank's ``ui`` rows, "seen" = their
        union with its ``val`` and ``test`` rows, transposed to item rows."""
        if exclude not in EXCLUDE:
            raise ValueError(f"exclude must be one of {EXCLUDE}, not {exclude!r}")
        pair = lambda b: (b.indptr, b.indices)
        rows = pair(sh.train_rows())
        if exclude == "seen":
            rows = union_csr(rows, pair(sh.held("val")), pair(sh.held("test")))
        return cls(transpose_csr(*rows, sh.n_items), sh.part["user"], sh.part["item"], sh.rank, k, group, device)

    @classmethod
    def from_rows(cls, train_items, test_set, val_set, n_users: int, n_items: int, part_u: RowPartition, part_i: RowPartition,
                  rank: int, k: int, exclude: str = "train", group=None, device="cuda") -> "ShardedAudience":
        """From the reference's dicts; every rank keeps the exclusion of its user block."""
        if part_u.n != int(n_users) or part_i.n != int(n_items):
            raise ValueError(f"{n_users} x {n_items} does not match the partitions ({part_u.n} x {part_i.n} rows)")
        rows = _block_rows(exclusion_rows(train_items, test_set, val_set, exclude), part_u, rank)
        return cls(transpose_csr(*rows, n_items), part_u, part_i, rank, k, group, device)

    def check_items(self, items) -> np.ndarray:
        ids = _host_ids(items)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= self.n_items):
            raise ValueError(_BAD_ITEM)
        return ids

    def gather_items(self, i_local: torch.Tensor) -> torch.Tensor:
        """Collective.  [block, d] item rows of every rank -> the full [n_items, d] table."""
        return all_gather_rows(i_local.detach(), self.pi, self.group)

    def exchange(self, send: torch.Tensor, send_rows: Sequence[int], recv_rows: Sequence[int]) -> torch.Tensor:
        """Collective.  Rows of `send`, in blocks of send_rows[r] rows for rank r, to their ranks; returns the rows received, in
        blocks of recv_rows[r] rows from rank r, in rank order."""
        if self.pu.world == 1:
            return send
        out = torch.empty(int(sum(recv_rows)), send.shape[1], dtype=send.dtype, device=send.device)
        dist.all_to_all_single(out, send.contiguous(), list(map(int, recv_rows)), list(map(int, send_rows)), group=self.group)
        return out

    def local(self, u_local: torch.Tensor) -> Recommender:
        """The ranker of this rank's real user rows (local ids) against item queries."""
        if u_local.shape[0] != self.pu.block:
            raise ValueError(f"a rank's user table holds {self.pu.block} rows (padded block), not {u_local.shape[0]}")
        return Recommender(u_local.detach()[:self.n_real], self.exclude, self.k)

    def mine(self, ids: np.ndarray) -> np.ndarray:
        """Positions in `ids` of the items in this rank's block."""
        return np.nonzero(ids // self.pi.block == self.rank_id)[0]

    def _chunk(self, rec: Recommender, ia: torch.Tensor, ids: np.ndarray):
        """Collective.  Steps 1-3 for the chunk `ids` (the same on every rank): (ids [m, k] int32, scores [m, k] fp32) of the m
        items of the chunk this rank owns, in their listed order."""
        k, world = self.k, self.pu.world
        owner = ids // self.pi.block
        order = np.argsort(owner, kind="stable")            # the rows for rank r form one block, in listed order
        send_rows = np.bincount(owner, minlength=world)
        n = ids.size
        part = torch.empty(n, 2 * k, dtype=torch.int32, device=self.device)     # per row: user ids, then the scores' bits
        if n:
            rec._launch(ia, torch.from_numpy(ids[order]).to(self.device), n, part, part[:, k:].view(torch.float32), 2 * k)
            if self.base:
                got = part[:, :k]
                got.copy_(torch.where(got >= 0, got + self.base, got))
        m = int(send_rows[self.rank_id])
        recv = self.exchange(part, send_rows.tolist(), [m] * world)
        out_ids = torch.empty(m, k, dtype=torch.int32, device=self.device)
        out_sc = torch.empty(m, k, dtype=torch.float32, device=self.device)
        merge_lists(recv, recv[:, k:].view(torch.float32), m, world, k, 2 * k, m * 2 * k, out_ids, out_sc, k)
        return out_ids, out_sc

    def _run(self, u_local: torch.Tensor, i_local: torch.Tensor, ids: np.ndarray, chunk: int):
        """Collective.  Yields (first position of the chunk's own rows among this rank's rows, ids, scores) chunk by chunk."""
        if chunk < 1:
            raise ValueError("chunk must be >= 1")
        rec = self.local(u_local)
        ia = rec._user_table(self.gather_items(i_local))
        done = 0
        for s in range(0, ids.size, chunk):
            got_ids, got_sc = self._chunk(rec, ia, ids[s:s + chunk])
            yield done, got_ids, got_sc
            done += got_ids.shape[0]

    def topk(self, u_local: torch.Tensor, i_local: torch.Tensor, items, chunk: int = 1 << 16):
        """Collective.  (ids [m, k] int64 user ids, scores [m, k] fp32, positions [m] host int64): the lists of the m listed items
        that are in this rank's item block, and where they stand in `items`."""
        ids = self.check_items(items)
        parts = [(i, s) for _, i, s in self._run(u_local, i_local, ids, chunk)]
        got_ids = torch.cat([p[0] for p in parts]) if parts else torch.empty(0, self.k, dtype=torch.int32, device=self.device)
        got_sc = torch.cat([p[1] for p in parts]) if parts else torch.empty(0, self.k, dtype=torch.float32, device=self.device)
        return got_ids.to(torch.int64), got_sc, self.mine(ids)

    def export(self, u_local: torch.Tensor, i_local: torch.Tensor, items, out_dir: str, chunk: int = 1 << 16) -> int:
        """Collective.  Writes ``rankRRRRR-of-WWWWW.{ids,scores,items}.npy`` with the lists of this rank's items, in their listed
        order, and commits them with ``rankRRRRR-of-WWWWW.json`` (ShardedRecommender.export's file logic and shared export id).
        Returns the number of rows written."""
        ids = self.check_items(items)
        prefix = _rank_prefix(self.rank_id, self.pi.world)
        stale = _sharded_stale(out_dir, self.rank_id, self.pi.world)
        export_id = shared_export_id(self.rank_id, self.pi.world, self.device, self.group)
        mine = ids[self.mine(ids)]
        files = _Files(out_dir, prefix, mine.size, self.k, export_id, stale, "items", _meta())
        try:
            if mine.size:
                files.arr["items"][:] = mine
            for s, got_ids, got_sc in self._run(u_local, i_local, ids, chunk):
                m = got_ids.shape[0]
                if m:
                    files.arr["ids"][s:s + m] = got_ids.cpu().numpy()
                    files.arr["scores"][s:s + m] = got_sc.cpu().numpy()
            files.commit()
        except BaseException:
            files.discard()
            raise
        return mine.size
