"""Similar items: the top-k nearest catalogue items of every item, by cosine similarity in one of three spaces, on the device with
no [items x items] score matrix anywhere.

  "model"            the eval-mode final item table i_f (what ``Trainer.test`` and ``recommend`` score against): collaborative
  "image" / "text"   the eval-mode modality projections Xv = Fv Wv^T + bv, Xt = Ft Wt^T + bt (Models.py:173-174, no dropout):
                     content.  A projection depends only on the item's own features, so it answers equally for items with many,
                     few or no interactions, and for the feature rows of items that are not in the catalogue.

  ``SimilarItems(table, k)``     one GPU: ``topk(items)`` -> (ids [n, k] int64, scores [n, k] fp32) on the device; ``export(items,
                                 out_dir)`` ranks the items chunk by chunk into ``ids.npy`` / ``scores.npy`` / ``items.npy``;
                                 ``topk_features`` / ``export_features`` rank the projected feature rows of new items.
  ``ShardedSimilarItems``        a row-sharded model (rowshard_step.py) on the ranks that hold it: every rank gathers the unit table
                                 once and ranks the listed items of its own block; ``export`` writes rankRRRRR-of-WWWWW.* per rank.
  ``read(out_dir)``              (items, ids, scores) of either layout.

Score: the dot product of unit rows x / max(|x|, 1e-12) (``mmssl_unit_rows``, F.normalize); a zero row stays zero, so all its
scores are 0 and its list holds the lowest ids.  Ranking: ``mmssl_recommend_topk`` unchanged, the unit table being both the query
and the candidate table -- best score first, equal scores lower item id first, -1 (score 0) past the end of a short list.  A
catalogue item never appears in its own list (an identity exclusion CSR, row r = [r]: 16 bytes per item), so with k >= n_items a
list has n_items - 1 entries; a feature row is ranked against the whole catalogue (an empty CSR).  Exports share recommend.py's
file logic (temporary names, renames, a manifest written last) with ``items.npy`` for the query ids; the manifest records the
space, and each of recommend.read / similar.read refuses the other's directories."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, ops
from .engine import P_WT, P_WV, Engine, FeatureStore
from .parallel import RowPartition, all_gather_rows
from .recommend import (MANIFEST, Recommender, _host_ids, _manifests, _new_export_id, _rank_prefix, _read, _sharded_stale,
                        shared_export_id)

SPACES = ("model", "image", "text")
FORMAT = "mmssl_b200.similar.v1"
_BAD_ITEM = "items holds an id outside [0, n_items)"


def _check_space(space: str) -> None:
    if space not in SPACES:
        raise ValueError(f"space must be one of {SPACES}, not {space!r}")


def identity_csr(n: int, device, base: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exclusion CSR of n rows, row r = [base + r]: every catalogue item is excluded from its own list."""
    return (torch.arange(n + 1, dtype=torch.int64, device=device),
            torch.arange(base, base + n, dtype=torch.int64, device=device))


def empty_csr(n: int, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exclusion CSR of n empty rows (its one index is never read: the ranking kernel takes a non-null index array)."""
    return torch.zeros(n + 1, dtype=torch.int64, device=device), torch.zeros(1, dtype=torch.int64, device=device)


def _meta(space: str, queries: str) -> dict:
    """The manifest fields of a similar-items export (one-GPU and row-sharded layouts alike)."""
    return dict(format=FORMAT, kind="similar", space=space, queries=queries)


def _check_feature_widths(P, image_dim: int, text_dim: int) -> None:
    """Feature rows must have the widths the projection weights were trained on: the tensor-core GEMM reads k = the rows' width
    columns of W, so narrower rows would be projected with a truncated W, silently."""
    want = (int(P[P_WV].shape[1]), int(P[P_WT].shape[1]))
    if (int(image_dim), int(text_dim)) != want:
        raise ValueError(f"feature rows of widths image {image_dim} / text {text_dim}: the model's projections take image {want[0]} "
                         f"/ text {want[1]}")


def _row_table(table: torch.Tensor, what: str) -> torch.Tensor:
    """A 2-D fp32 CUDA table as the row kernels read it: unit column stride, row stride % 4 == 0, 16-byte aligned (a copy if not)."""
    t = table.detach()
    if t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2:
        raise TypeError(f"{what} must be a 2-D fp32 CUDA tensor")
    if t.stride(1) != 1 or t.stride(0) % 4 or t.data_ptr() % 16:
        t = t.contiguous().clone()
    return t


def project(engine: Engine, P, feats: Sequence[FeatureStore], plan_rows: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(Xv, Xt) [n, d] of the feature rows `feats` (image, text): the eval-mode projection, through the forward's own grouped
    launch, with no dropout mask.  plan_rows: see Engine._project (the catalogue's item count makes new rows project with the
    catalogue's bits).  Feature widths other than the weights' are refused."""
    d, n = engine.d, feats[0].n_items
    if feats[1].n_items != n:
        raise ValueError(f"{n} image rows and {feats[1].n_items} text rows")
    _check_feature_widths(P, feats[0].dim, feats[1].dim)
    x = torch.empty(n, 2 * d, dtype=torch.float32, device=P["image_trans.weight"].device)
    xv, xt = x[:, :d], x[:, d:]
    if n:
        engine._project(P, feats, (None, None), (xv, xt), plan_rows=plan_rows)
    return xv, xt


def space_table(engine: Engine, P, feats: Sequence[FeatureStore], graphs, space: str) -> torch.Tensor:
    """The [n_items, d] table of a space for a model's parameters P, feature stores and the six graphs of ``Engine.forward``:
    the eval-mode i_f for "model", the eval-mode projection for "image" / "text"."""
    _check_space(space)
    if space == "model":
        outs, _ = engine.forward(P, feats, graphs, None, want_sumsq=False)        # model.eval(): no dropout
        return outs[1]
    return project(engine, P, feats)[0 if space == "image" else 1]


def _feature_rows(rows) -> torch.Tensor:
    f = torch.as_tensor(np.asarray(rows, np.float32) if not torch.is_tensor(rows) else rows)
    if f.dim() != 2:
        raise ValueError("feature rows must be a 2-D array")
    return f


class SimilarItems:
    """Top-k similar catalogue items against one [n_items, d] table (any of the three spaces; ``from_model`` builds it).
    ``engine`` / ``P``: the model the table was projected with, needed only by the feature queries of "image" / "text"."""

    def __init__(self, table: torch.Tensor, k: int, space: str = "model", engine: Optional[Engine] = None, P=None):
        _lib.load(require_device=True)
        _check_space(space)
        t = _row_table(table, "the table")
        self.unit = ops.unit_rows(t)
        self.n_items, self.d, self.space, self.device = t.shape[0], t.shape[1], space, t.device
        self.rec = Recommender(self.unit, identity_csr(self.n_items, self.device), k)
        self.k = self.rec.k
        self.engine, self.P = engine, P

    @classmethod
    def from_model(cls, engine: Engine, P, feats: Sequence[FeatureStore], graphs, k: int, space: str = "model") -> "SimilarItems":
        return cls(space_table(engine, P, feats, graphs, space), k, space, engine, P)

    def meta(self, queries: str = "catalogue") -> dict:
        return _meta(self.space, queries)

    def check_items(self, items) -> np.ndarray:
        ids = _host_ids(items)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= self.n_items):
            raise ValueError(_BAD_ITEM)
        return ids

    def topk(self, items) -> Tuple[torch.Tensor, torch.Tensor]:
        """(ids [n, k] int64, scores [n, k] fp32) on the device, row i for items[i]; n == 0 launches nothing."""
        return self.rec.topk(self.unit, self.check_items(items))

    def export(self, items, out_dir: str, chunk: int = 1 << 16) -> int:
        """Ranks `items` ``chunk`` at a time into ``ids.npy`` (int32 [n, k]), ``scores.npy`` (fp32 [n, k]) and ``items.npy`` (int64
        [n]) in out_dir and commits them with ``manifest.json`` (recommend.Recommender.export's file logic).  Returns n."""
        ids = self.check_items(items)
        _, ranks = _manifests(out_dir)
        return self.rec._export(self.unit, ids, ids, out_dir, chunk, "", _new_export_id(), [MANIFEST] + list(ranks.values()),
                                "items", self.meta())

    # ---- feature rows of items that are not in the catalogue
    def _feature_queries(self, image_feats, text_feats) -> Tuple[torch.Tensor, Recommender]:
        if self.space == "model":
            raise ValueError('feature queries need space "image" or "text": the "model" table has no row for a new item')
        if self.engine is None:
            raise ValueError("feature queries need the model the table was projected with (SimilarItems.from_model)")
        img, txt = _feature_rows(image_feats), _feature_rows(text_feats)
        _check_feature_widths(self.P, img.shape[1], txt.shape[1])       # before the rows are split and copied to the device
        feats = tuple(FeatureStore(f.to(device=self.device, dtype=torch.float32).contiguous()) for f in (img, txt))
        x = project(self.engine, self.P, feats, plan_rows=self.n_items)[0 if self.space == "image" else 1]
        m = x.shape[0]
        return ops.unit_rows(x), Recommender(self.unit, empty_csr(m, self.device), self.k)

    def topk_features(self, image_feats, text_feats) -> Tuple[torch.Tensor, torch.Tensor]:
        """The lists of m new items given by their feature rows (image [m, Dv], text [m, Dt]: the projection takes both; the
        table's space picks one): projected with the trained weights, ranked against the whole catalogue, nothing excluded."""
        q, rec = self._feature_queries(image_feats, text_feats)
        return rec.topk(q, np.arange(q.shape[0], dtype=np.int64))

    def export_features(self, image_feats, text_feats, out_dir: str, chunk: int = 1 << 16) -> int:
        """``topk_features`` exported like ``export``; ``items.npy`` holds the row numbers of the feature rows."""
        q, rec = self._feature_queries(image_feats, text_feats)
        rows = np.arange(q.shape[0], dtype=np.int64)
        _, ranks = _manifests(out_dir)
        return rec._export(q, rows, rows, out_dir, chunk, "", _new_export_id(), [MANIFEST] + list(ranks.values()), "items",
                           self.meta("features"))


def read(out_dir: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(items [n] int64, ids [n, k] int32, scores [n, k] fp32) of the committed similar-items export in out_dir, either layout
    (recommend.read's rules: rank files in ascending item order, an incomplete row-sharded export refused); a recommendation
    export is refused."""
    return _read(out_dir, "items", FORMAT, "similar-items")


class ShardedSimilarItems:
    """``SimilarItems`` of a model whose item table is row-sharded over the ranks of a process group (rowshard_step.py): one per
    rank.  ``topk`` / ``export`` take the rank's padded [block, d] item rows of the space (``RowShardedHotStep.final_embeddings``'s
    i_f for "model", ``RowShardedHotStep.projections`` for "image" / "text") and the same list of global item ids on every rank.
    Every rank computes the unit rows of its block, all-gathers the unit table once (padding dropped: a padding row is never a
    candidate) and ranks the listed items of its block (never a padding row) with an identity exclusion of global ids.  A unit
    row depends only on its row, so every list is bitwise the one-GPU ``SimilarItems``'s on the gathered table; each rank returns
    and writes its own lists only."""

    def __init__(self, part_i: RowPartition, rank: int, k: int, space: str = "model", group=None, device="cuda"):
        _check_space(space)
        self.pi, self.rank_id, self.k, self.space, self.group = part_i, int(rank), int(k), space, group
        if self.k < 1:
            raise ValueError("k must be >= 1")
        self.n_items, self.device = part_i.n, torch.device(device)

    def check_items(self, items) -> np.ndarray:
        ids = _host_ids(items)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= self.n_items):
            raise ValueError(_BAD_ITEM)
        return ids

    def gather(self, unit_local: torch.Tensor) -> torch.Tensor:
        """Collective.  [block, d] unit rows of every rank -> the [n_items, d] unit table."""
        return all_gather_rows(unit_local, self.pi, self.group)

    def local(self, table_local: torch.Tensor) -> Tuple[torch.Tensor, Recommender]:
        """Collective.  (the unit rows of this rank's block, the recommender of the block's rows against the gathered table)."""
        if table_local.shape[0] != self.pi.block:
            raise ValueError(f"a rank's table holds {self.pi.block} rows (padded block), not {table_local.shape[0]}")
        unit_local = ops.unit_rows(_row_table(table_local, "a rank's table"))
        return unit_local, Recommender(self.gather(unit_local), identity_csr(self.pi.block, self.device, self.rank_id * self.pi.block),
                                       self.k)

    def export_id(self) -> int:
        """Collective.  A fresh random id, the same on every rank."""
        return shared_export_id(self.rank_id, self.pi.world, self.device, self.group)

    def mine(self, ids: np.ndarray) -> np.ndarray:
        """Positions in `ids` of the items in this rank's block."""
        return np.nonzero(ids // self.pi.block == self.rank_id)[0]

    def topk(self, table_local: torch.Tensor, items):
        """Collective.  (ids [m, k] int64, scores [m, k] fp32, positions [m] host int64): the lists of the m listed items that are in
        this rank's block, and where they stand in `items`."""
        ids = self.check_items(items)
        unit_local, rec = self.local(table_local)
        pos = self.mine(ids)
        got_ids, got_sc = rec.topk(unit_local, ids[pos] - self.rank_id * self.pi.block)
        return got_ids, got_sc, pos

    def export(self, table_local: torch.Tensor, items, out_dir: str, chunk: int = 1 << 16) -> int:
        """Collective.  Writes ``rankRRRRR-of-WWWWW.{ids,scores,items}.npy`` with this rank's items, in their listed order, and
        commits them with ``rankRRRRR-of-WWWWW.json`` (ShardedRecommender.export's file logic).  Returns the rows written."""
        ids = self.check_items(items)
        prefix = _rank_prefix(self.rank_id, self.pi.world)
        stale = _sharded_stale(out_dir, self.rank_id, self.pi.world)
        export_id = self.export_id()
        unit_local, rec = self.local(table_local)
        mine = ids[self.mine(ids)]
        return rec._export(unit_local, mine - self.rank_id * self.pi.block, mine, out_dir, chunk, prefix, export_id, stale, "items",
                           _meta(self.space, "catalogue"))
