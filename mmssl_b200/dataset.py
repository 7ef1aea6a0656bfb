"""On-disk formats (SURVEY 8f "next" #4, second half).

1. ``ReferenceDataset.load(dir)`` reads the reference's dataset directory exactly like ``utility/load_data.py:Data.__init__``
   (:10-88) and ``Trainer.__init__`` (main.py:54-58): ``train.json`` / ``val.json`` / ``test.json`` (user -> item list),
   ``train_mat`` (pickled scipy CSR), ``image_feat.npy`` / ``text_feat.npy``; same inference of n_users / n_items, same
   ``exist_users`` order, same ``train_items`` / ``test_set`` / ``val_set`` dictionaries.
2. ``write_shards`` converts it ONCE into flat little-endian arrays: the four normalised operands the propagation needs
   (A_ui, A_iu and their transposes, csr_norm(mean_flag=True) of main.py:89-103) as CSR ``indptr.i64 / indices.i32 /
   values.f32`` and the two feature matrices row-major fp32.
3. ``ShardedDataset.open(dir, rank, world)`` memory-maps them and hands every rank only ITS row blocks (parallel.RowPartition:
   user rows of A_ui and (A_iu)^T, item rows of A_iu, (A_ui)^T and of the features) without reading the rest: the slices are
   views of the maps (indices / values are contiguous per row block), so a rank touches 1/world of the bytes and the
   host->device copy can run straight from the page cache.
4. The held-out sets (``val_set`` / ``test_set``) are written beside the operands as CSR over users (``val.*`` / ``test.*``:
   sorted rows, global item ids, empty rows for users without one); ``ShardedDataset.held`` and ``train_rows`` hand a rank the
   rows of its user block for the sharded evaluator (evaluate.ShardedEvaluator).  A directory written before they existed
   still opens and trains; only ``held`` needs them.
"""
from __future__ import annotations

import itertools
import json
import os
import pickle
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import scipy.sparse as sp

from .parallel import RowPartition
from .synthetic import csr_norm

OPERANDS = ("ui", "iu", "iuT", "uiT")       # A_ui [U,I], A_iu [I,U], (A_iu)^T [U,I], (A_ui)^T [I,U]
ROW_SPACE = {"ui": "user", "iuT": "user", "iu": "item", "uiT": "item"}
HELD = ("val", "test")                      # held-out sets, CSR over users (meta.json "held")


@dataclass
class ReferenceDataset:
    n_users: int
    n_items: int
    n_train: int
    n_test: int
    exist_users: List[int]
    train_items: Dict[int, List[int]]
    test_set: Dict[int, List[int]]
    val_set: Dict[int, List[int]]
    train_mat: sp.csr_matrix
    image_feats: np.ndarray
    text_feats: np.ndarray
    path: str = field(default="", repr=False)

    @classmethod
    def load(cls, path: str, mmap_features: bool = True) -> "ReferenceDataset":
        def read(name):
            with open(os.path.join(path, name)) as f:
                return json.load(f)
        train, test, val = read("train.json"), read("test.json"), read("val.json")
        n_users = n_items = n_train = n_test = 0
        exist_users: List[int] = []
        for uid, items in train.items():                        # load_data.py:30-37
            if len(items) == 0:
                continue
            uid = int(uid)
            exist_users.append(uid)
            n_items = max(n_items, max(items))
            n_users = max(n_users, uid)
            n_train += len(items)
        for uid, items in test.items():                         # :39-45 (empty lists are skipped by the bare except)
            if len(items):
                n_items = max(n_items, max(items))
                n_test += len(items)
        for uid, items in val.items():                          # :47-53 (only the n_items update survives there)
            if len(items):
                n_items = max(n_items, max(items))
        n_items += 1
        n_users += 1
        keep = lambda d: {int(u): list(its) for u, its in d.items() if len(its)}      # :62-88
        with open(os.path.join(path, "train_mat"), "rb") as f:  # main.py:58 (the reference's own format is a pickle)
            train_mat = pickle.load(f).tocsr()
        mode = "r" if mmap_features else None
        return cls(n_users, n_items, n_train, n_test, exist_users, keep(train), keep(test), keep(val), train_mat,
                   np.load(os.path.join(path, "image_feat.npy"), mmap_mode=mode),
                   np.load(os.path.join(path, "text_feat.npy"), mmap_mode=mode), path)


def _write(path: str, arr: np.ndarray, dtype) -> None:
    np.ascontiguousarray(arr, dtype=np.dtype(dtype).newbyteorder("<")).tofile(path)


def held_csr(rows: Dict[int, List[int]], n_rows: int) -> Tuple[np.ndarray, np.ndarray]:
    """dict user -> item list -> CSR (indptr int64 [n_rows + 1], indices int64) with every row sorted and duplicate ids kept,
    the rows ``evaluate.Evaluator`` builds from the same dict."""
    users = np.fromiter((int(u) for u in rows), np.int64, len(rows))
    if users.size and (users.min() < 0 or users.max() >= n_rows):
        raise ValueError(f"held-out rows name a user outside [0, {n_rows})")
    lens = np.fromiter((len(v) for v in rows.values()), np.int64, len(rows))
    indptr = np.zeros(n_rows + 1, np.int64)
    indptr[users + 1] = lens
    np.cumsum(indptr, out=indptr)
    flat = np.fromiter(itertools.chain.from_iterable(rows.values()), np.int64, int(lens.sum()))
    return indptr, flat[np.lexsort((flat, np.repeat(users, lens)))]


def write_shards(ds: ReferenceDataset, out_dir: str) -> Dict[str, object]:
    """Flat arrays + meta.json.  Independent of the world size: the row blocks are cut at open time."""
    os.makedirs(out_dir, exist_ok=True)
    R = ds.train_mat.astype(np.float32).tocsr()
    U, I = R.shape
    a_ui, a_iu = csr_norm(R), csr_norm(R.T.tocsr())
    mats = {"ui": a_ui, "iu": a_iu, "iuT": a_iu.T.tocsr(), "uiT": a_ui.T.tocsr()}
    meta = {"format": "mmssl_b200.shards.v1", "n_users": int(U), "n_items": int(I), "operands": {},
            "image_dim": int(ds.image_feats.shape[1]), "text_dim": int(ds.text_feats.shape[1])}
    for name, m in mats.items():
        m.sort_indices()
        _write(os.path.join(out_dir, f"{name}.indptr.i64"), m.indptr, np.int64)
        _write(os.path.join(out_dir, f"{name}.indices.i32"), m.indices, np.int32)
        _write(os.path.join(out_dir, f"{name}.values.f32"), m.data, np.float32)
        meta["operands"][name] = {"rows": int(m.shape[0]), "cols": int(m.shape[1]), "nnz": int(m.nnz)}
    _write(os.path.join(out_dir, "image_feat.f32"), ds.image_feats, np.float32)
    _write(os.path.join(out_dir, "text_feat.f32"), ds.text_feats, np.float32)
    meta["held"] = {}
    for name, rows in (("val", ds.val_set), ("test", ds.test_set)):
        indptr, indices = held_csr(rows, U)
        _write(os.path.join(out_dir, f"{name}.indptr.i64"), indptr, np.int64)
        _write(os.path.join(out_dir, f"{name}.indices.i32"), indices, np.int32)
        meta["held"][name] = {"rows": int(U), "nnz": int(indices.size)}
    with open(os.path.join(out_dir, "meta.json"), "w") as f:
        json.dump(meta, f, indent=1)
    return meta


@dataclass
class CsrBlock:
    """Row block [lo, hi) of an operand, padded to `block` rows; indptr is rebased to 0, indices are GLOBAL column ids.
    ``values`` is None for a pattern (held-out rows, training rows): ``to_scipy`` then gives it ones."""
    indptr: np.ndarray
    indices: np.ndarray
    values: Optional[np.ndarray]
    shape: Tuple[int, int]
    lo: int
    hi: int

    def to_scipy(self) -> sp.csr_matrix:
        vals = self.values if self.values is not None else np.ones(self.indices.size, np.float32)
        return sp.csr_matrix((vals, self.indices, self.indptr), shape=self.shape)


class ShardedDataset:
    def __init__(self, root: str, rank: int, world: int):
        with open(os.path.join(root, "meta.json")) as f:
            self.meta = json.load(f)
        if self.meta.get("format") != "mmssl_b200.shards.v1":
            raise ValueError(f"{root}: not a mmssl_b200 shard directory")
        self.root, self.rank, self.world = root, rank, world
        self.n_users, self.n_items = self.meta["n_users"], self.meta["n_items"]
        self.part = {"user": RowPartition(self.n_users, world), "item": RowPartition(self.n_items, world)}

    @classmethod
    def open(cls, root: str, rank: int = 0, world: int = 1) -> "ShardedDataset":
        return cls(root, rank, world)

    def _map(self, name: str, dtype, shape=None) -> np.ndarray:
        return np.memmap(os.path.join(self.root, name), dtype=np.dtype(dtype).newbyteorder("<"), mode="r", shape=shape)

    def _block(self, name: str, part: RowPartition, rows: int, nnz: int, cols: int, values: bool) -> CsrBlock:
        lo, hi = part.bounds(self.rank)
        ip = self._map(f"{name}.indptr.i64", np.int64, (rows + 1,))
        b, e = int(ip[lo]), int(ip[hi])
        indptr = np.empty(part.block + 1, np.int64)
        indptr[:hi - lo + 1] = ip[lo:hi + 1] - b
        indptr[hi - lo + 1:] = e - b                             # padding rows are empty
        if nnz == 0:                                             # an empty file cannot be mapped (an empty held-out set)
            return CsrBlock(indptr, np.zeros(0, np.int32), np.zeros(0, np.float32) if values else None, (part.block, cols), lo, hi)
        idx = self._map(f"{name}.indices.i32", np.int32, (nnz,))[b:e]
        val = self._map(f"{name}.values.f32", np.float32, (nnz,))[b:e] if values else None
        return CsrBlock(indptr, idx, val, (part.block, cols), lo, hi)

    def operand(self, name: str) -> CsrBlock:
        info = self.meta["operands"][name]
        return self._block(name, self.part[ROW_SPACE[name]], info["rows"], info["nnz"], info["cols"], True)

    def train_rows(self) -> CsrBlock:
        """The training items of the rank's user block: the column pattern of its ``ui`` rows (sorted global item ids, no
        values), i.e. the rows of ``train_mat`` -- the graph the model trains on, and ``Data.train_items`` wherever the
        dataset's train.json and train_mat agree."""
        info = self.meta["operands"]["ui"]
        return self._block("ui", self.part["user"], info["rows"], info["nnz"], info["cols"], False)

    def held(self, split: str) -> CsrBlock:
        """The held-out items ('val' or 'test') of the rank's user block: sorted global item ids, no values."""
        if split not in HELD:
            raise ValueError(f"split must be one of {HELD}, not {split!r}")
        info = self.meta.get("held", {}).get(split)
        if info is None:
            raise ValueError(f"{self.root}: no held-out '{split}' rows ({split}.indptr.i64 / {split}.indices.i32 are missing; "
                             f"write the directory again with dataset.write_shards)")
        return self._block(split, self.part["user"], info["rows"], info["nnz"], self.n_items, False)

    def features(self, which: str) -> np.ndarray:
        """This rank's item rows of 'image' / 'text' features: a [hi-lo, D] view of the map (no copy)."""
        dim = self.meta[f"{which}_dim"]
        lo, hi = self.part["item"].bounds(self.rank)
        return self._map(f"{which}_feat.f32", np.float32, (self.n_items, dim))[lo:hi]

    def bytes_touched(self) -> int:
        """Bytes this rank maps for its blocks (what a cold open reads from disk)."""
        n = 0
        for name in OPERANDS:
            blk = self.operand(name)
            n += blk.indptr.nbytes + blk.indices.nbytes + blk.values.nbytes
        return n + self.features("image").nbytes + self.features("text").nbytes
