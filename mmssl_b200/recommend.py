"""Recommendations of a trained model: the top-k items each user has not seen, on the device, with no [users x items] score
matrix anywhere (``mmssl_recommend_topk``: the evaluation sweep of csrc/eval.cu in its recommendation mode).

  ``Recommender(item_table, exclude, k)``     one GPU: ``topk(user_table, users)`` -> (ids [n, k] int64, scores [n, k] fp32) on the
                                              device; ``export(user_table, users, out_dir)`` ranks the users chunk by chunk into
                                              ``ids.npy`` / ``scores.npy`` / ``users.npy``.
  ``ShardedRecommender``                      a row-sharded model (rowshard_step.py) on the ranks that hold it: every rank gathers
                                              the item table once and ranks the listed users of its own user block; ``export``
                                              writes ``rankRRRRR-of-WWWWW.{ids,scores,users}.npy`` per rank.
  ``read(out_dir)``                           (users, ids, scores) of either layout.

Ranking: best score first, equal scores lower item id first, items of the user's ``exclude`` row dropped, -1 (score 0) past the
end of a list shorter than k.  Two exclusion sets (``exclusion_rows``): "train" -- the training rows, what ``Trainer.test`` masks,
so the lists are ``Evaluator.rank``'s ranked / ranked_scores with Ks = [k], bit for bit -- and "seen" -- train, val and test,
what serving wants.  Every file is written under a temporary name and renamed into place once complete (as checkpoint.save does),
and an export is committed by a small manifest written last (``manifest.json``, or ``rankRRRRR-of-WWWWW.json`` per rank with an
export id shared by the ranks); ``read`` reads committed exports only, so an interrupted export, or a row-sharded one that did not
finish on every rank, is never read, alone or mixed with the files of an earlier export in the same directory."""
from __future__ import annotations

import json
import os
import re
import tempfile
from typing import Mapping, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from ._lib import ptr, stream
from .evaluate import _BAD_USER, _block_rows, _device_csr, _rows_to_csr
from .parallel import RowPartition, all_gather_rows

EXCLUDE = ("train", "seen")
FILES = ("ids", "scores", "users")
FORMAT = "mmssl_b200.recommend.v1"
QUERY_FILES = ("users", "items", "queries")   # the row-id file of a recommendation / similar-items or audience / fold-in export
MANIFEST = "manifest.json"
_RANK_MANIFEST = re.compile(r"rank(\d{5})-of-(\d{5})\.json")


def exclusion_rows(train_items: Mapping[int, Sequence[int]], test_set: Mapping[int, Sequence[int]],
                   val_set: Mapping[int, Sequence[int]], which: str) -> Mapping[int, Sequence[int]]:
    """dict user -> items a user must not be shown: "train" the training rows, "seen" train | val | test without duplicates."""
    if which not in EXCLUDE:
        raise ValueError(f"exclude must be one of {EXCLUDE}, not {which!r}")
    if which == "train":
        return train_items
    seen = {}
    for rows in (train_items, val_set, test_set):
        for u, its in rows.items():
            seen.setdefault(int(u), set()).update(int(i) for i in its)
    return {u: sorted(s) for u, s in seen.items()}


def union_csr(*blocks) -> Tuple[np.ndarray, np.ndarray]:
    """Row-wise union of CSR blocks with the same row count ((indptr, indices) host arrays): sorted rows, no duplicates."""
    n = len(blocks[0][0]) - 1
    rows = np.concatenate([np.repeat(np.arange(n, dtype=np.int64), np.diff(np.asarray(ip, np.int64))) for ip, _ in blocks])
    cols = np.concatenate([np.asarray(ix, np.int64)[int(ip[0]):int(ip[-1])] for ip, ix in blocks])
    width = int(cols.max()) + 1 if cols.size else 1
    key = np.unique(rows * width + cols)                # sorted by (row, item), duplicates dropped
    r, c = key // width, key % width
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(r, minlength=n), out=indptr[1:])
    return indptr, c


def _host_ids(users) -> np.ndarray:
    ids = users.detach().cpu().numpy() if torch.is_tensor(users) else users
    return np.ascontiguousarray(np.asarray(ids, np.int64).reshape(-1))     # (torch.from_numpy takes no negative strides)


def _tmp_path(path: str) -> str:
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(path) + ".", suffix=".tmp", dir=os.path.dirname(path))
    os.close(fd)
    return tmp


def _manifest_name(prefix: str) -> str:
    """The manifest of the files ``<prefix>{ids,scores,users}.npy``: manifest.json, or rankRRRRR-of-WWWWW.json."""
    return prefix + "json" if prefix else MANIFEST


def _manifests(out_dir: str) -> Tuple[bool, dict]:
    """(one-GPU manifest present, {(rank, world): name} of the rank manifests) in out_dir."""
    names = os.listdir(out_dir) if os.path.isdir(out_dir) else []
    ranks = {}
    for name in names:
        m = _RANK_MANIFEST.fullmatch(name)
        if m:
            ranks[(int(m.group(1)), int(m.group(2)))] = name
    return MANIFEST in names, ranks


class _Files:
    """The three output arrays of an export under temporary names in out_dir.  On creation the manifests this export supersedes
    are removed (from then on the directory holds no committed export that the new files could mix with); ``commit`` renames
    the files over their final names and then writes the export's manifest, which is what makes them readable."""

    def __init__(self, out_dir: str, prefix: str, n: int, k: int, export_id: int, stale, query: str = "users", meta=None):
        """query: the name of the file of row ids ("users" here, "items" for similar.py); meta: the manifest's format and
        whatever else it records (default: a recommendation export).  The other kind's row-id file under the same prefix is
        removed with the stale manifests: it belongs to an export this one supersedes and would be left behind."""
        os.makedirs(out_dir, exist_ok=True)
        stale = list(stale) + [f"{prefix}{q}.npy" for q in QUERY_FILES if q != query]
        for name in stale:
            try:
                os.remove(os.path.join(out_dir, name))
            except FileNotFoundError:
                pass
        self.files = ("ids", "scores", query)
        self.final = {f: os.path.abspath(os.path.join(out_dir, f"{prefix}{f}.npy")) for f in self.files}
        self.manifest = os.path.abspath(os.path.join(out_dir, _manifest_name(prefix)))
        self.meta = dict(meta or dict(format=FORMAT), export=int(export_id), n=int(n), k=int(k))
        self.tmp, self.arr = {}, {}
        spec = {"ids": (np.int32, (n, k)), "scores": (np.float32, (n, k)), query: (np.int64, (n,))}
        try:
            for f, (dt, shape) in spec.items():
                self.tmp[f] = _tmp_path(self.final[f])
                if n:
                    self.arr[f] = np.lib.format.open_memmap(self.tmp[f], mode="w+", dtype=dt, shape=shape)
                else:                                 # a zero-size array cannot be memory-mapped
                    with open(self.tmp[f], "wb") as fh:
                        np.save(fh, np.zeros(shape, dt))
        except BaseException:
            self.discard()
            raise

    def commit(self) -> None:
        for f in self.files:
            a = self.arr.pop(f, None)
            if a is not None:
                a.flush()
                del a
            with open(self.tmp[f], "rb+") as fh:
                os.fsync(fh.fileno())
        for f in self.files:
            os.replace(self.tmp[f], self.final[f])
        tmp = _tmp_path(self.manifest)
        try:
            with open(tmp, "w") as fh:
                json.dump(self.meta, fh)
                fh.flush()
                os.fsync(fh.fileno())
            os.replace(tmp, self.manifest)
        except BaseException:
            if os.path.exists(tmp):
                os.remove(tmp)
            raise

    def discard(self) -> None:
        self.arr.clear()
        for p in self.tmp.values():
            if os.path.exists(p):
                os.remove(p)


# Slicing of the candidates (Recommender._slices)
_SLICE_CTAS_PER_SM = 2              # CTAs per SM a launch should reach before it is left unsliced
_SLICE_MIN = 4096                   # candidates per slice at least: a shorter slice costs more in setup and merge than it saves
_SLICE_BYTES = 256 << 20            # device memory of the partial lists (ids and scores, slices x n x k) at most
_MAX_SLICES = 65535


def merge_lists(ids: torch.Tensor, scores: torch.Tensor, n: int, n_lists: int, k: int, ld: int, stride: int, out_ids: torch.Tensor,
                out_scores: torch.Tensor, ldo: int) -> None:
    """``mmssl_topk_merge``: the best k of n_lists sorted partial lists per row (entry i of list q of row r at element
    q * stride + r * ld + i of ids / scores) into rows of leading dimension ldo of out_ids / out_scores."""
    if n:
        _lib.check(_lib.load().mmssl_topk_merge(ptr(ids), ptr(scores), n, n_lists, k, ld, stride, ptr(out_ids), ptr(out_scores), ldo,
                                                stream()))


def _check_sorted_rows(indptr: torch.Tensor, indices: torch.Tensor) -> None:
    """The kernel finds excluded items by binary search in each row: an unsorted row would let excluded items through."""
    nnz = indices.numel()
    if nnz > 1:
        ok = indices[1:] >= indices[:-1]
        starts = indptr[1:-1]
        ok[starts[(starts > 0) & (starts < nnz)] - 1] = True       # a row may start below the previous row's last item
        if not bool(ok.all()):
            raise ValueError("the exclusion rows must be sorted (ascending item ids within each row)")


class Recommender:
    """Top-k unseen items against one item table.  ``exclude`` is (indptr [n_users + 1], indices) int64 on the table's device,
    sorted within each row (``from_rows`` builds it from the reference's dicts); its row count bounds the user ids."""

    def __init__(self, item_table: torch.Tensor, exclude: Tuple[torch.Tensor, torch.Tensor], k: int):
        _lib.load(require_device=True)
        ia = item_table.detach()
        if ia.dtype != torch.float32 or not ia.is_cuda or ia.dim() != 2:
            raise TypeError("the item table must be a 2-D fp32 CUDA tensor")
        if ia.stride(1) != 1 or ia.stride(0) % 4 or ia.data_ptr() % 16:
            ia = ia.contiguous().clone()
        self.items, self.n_items, self.d = ia, ia.shape[0], ia.shape[1]
        self.k = int(k)
        if self.k < 1:
            raise ValueError("k must be >= 1")
        ip, ix = exclude
        if ip.dtype != torch.int64 or ix.dtype != torch.int64 or ip.dim() != 1 or ix.dim() != 1 or ip.numel() < 1:
            raise TypeError("the exclusion CSR is two 1-D int64 tensors (indptr [n_users + 1], indices)")
        if ip.device != ia.device or ix.device != ia.device:
            raise ValueError(f"the exclusion CSR is on {ip.device} / {ix.device}, the item table on {ia.device}")
        _check_sorted_rows(ip, ix)
        self.exclude, self.n_users = (ip, ix), ip.numel() - 1
        self.device = ia.device
        self.sms = _lib.load().mmssl_sm_count()

    @classmethod
    def from_rows(cls, item_table: torch.Tensor, train_items, test_set, val_set, n_users: int, k: int,
                  exclude: str = "train") -> "Recommender":
        """From the reference's dicts (``Data.train_items`` / ``test_set`` / ``val_set``) and an exclusion set name."""
        return cls(item_table, _rows_to_csr(exclusion_rows(train_items, test_set, val_set, exclude), n_users, item_table.device), k)

    def check_users(self, users, n_rows: int) -> np.ndarray:
        ids = _host_ids(users)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= min(self.n_users, n_rows)):
            raise ValueError(_BAD_USER)
        return ids

    def _user_table(self, user_table: torch.Tensor) -> torch.Tensor:
        ua = user_table.detach()
        if ua.dtype != torch.float32 or not ua.is_cuda:
            raise TypeError("the user table must be an fp32 CUDA tensor")
        if ua.dim() != 2 or ua.shape[1] != self.d:
            raise ValueError(f"user table of width {ua.shape[-1]}, the item table's is {self.d}")
        return ua if ua.stride(1) == 1 else ua.contiguous()

    def _slices(self, n: int) -> int:
        """How many contiguous slices of the candidates a launch of n queries ranks separately (1: the unsliced sweep).  The sweep
        gives a CTA 8 queries and every candidate, so fewer than _SLICE_CTAS_PER_SM CTAs per SM leave SMs idle; slicing fills
        them, as long as a slice keeps at least _SLICE_MIN (and 8 k) candidates and the partial lists stay within _SLICE_BYTES.
        The merged lists are the unsliced lists bit for bit, so this choice changes the time of a call, never its result."""
        if n < 1:
            return 1
        tiles = -(-n // 8)
        want = -(-_SLICE_CTAS_PER_SM * self.sms // tiles)
        most = self.n_items // max(_SLICE_MIN, 8 * self.k)
        fits = _SLICE_BYTES // (8 * n * self.k)
        return max(1, min(want, most, fits, _MAX_SLICES))

    def _launch(self, ua, users_dev, n: int, ids, scores, ldo: int, key_ws=None) -> None:
        """Ranks users_dev[0, n) into ids / scores rows of leading dimension ldo (n > 0): one sweep, or a sliced sweep into
        partial lists and their merge (_slices).  key_ws: a workspace from _key_ws, replaced here when it is too small."""
        lib = _lib.load()
        s = self._slices(n)
        if key_ws is None or key_ws.numel() * 8 < self._ws_bytes(n, s):
            key_ws = self._key_ws(n)
        args = (ptr(ua), ua.stride(0), ptr(self.items), self.items.stride(0), self.n_items, self.d, ptr(users_dev), n,
                ptr(self.exclude[0]), ptr(self.exclude[1]), self.k)
        if s == 1:
            _lib.check(lib.mmssl_recommend_topk(*args, ldo, ptr(ids), ptr(scores), ptr(key_ws), stream()))
            return
        part_ids = torch.empty(s, n, self.k, dtype=torch.int32, device=self.device)
        part_sc = torch.empty(s, n, self.k, dtype=torch.float32, device=self.device)
        _lib.check(lib.mmssl_recommend_topk_sliced(*args, s, ptr(part_ids), ptr(part_sc), ptr(key_ws), stream()))
        merge_lists(part_ids, part_sc, n, s, self.k, self.k, n * self.k, ids, scores, ldo)

    def _ws_bytes(self, n: int, s: int) -> int:
        return _lib.load().mmssl_recommend_sliced_workspace_bytes(n, self.k, self.n_items, self.d, s)

    def _key_ws(self, n: int):
        nbytes = self._ws_bytes(n, self._slices(n))
        return torch.empty(nbytes // 8, dtype=torch.int64, device=self.device) if nbytes else None

    def topk(self, user_table: torch.Tensor, users) -> Tuple[torch.Tensor, torch.Tensor]:
        """(ids [n, k] int64, scores [n, k] fp32) on the device, row i for users[i]; n == 0 launches nothing."""
        ua = self._user_table(user_table)
        ids_np = self.check_users(users, ua.shape[0])
        n, dev = ids_np.size, self.device
        ids = torch.empty(n, self.k, dtype=torch.int32, device=dev)
        scores = torch.empty(n, self.k, dtype=torch.float32, device=dev)
        if n:
            self._launch(ua, torch.from_numpy(ids_np).to(dev), n, ids, scores, self.k)
        return ids.to(torch.int64), scores

    def export(self, user_table: torch.Tensor, users, out_dir: str, chunk: int = 1 << 16, prefix: str = "") -> int:
        """Ranks `users` ``chunk`` at a time into ``<prefix>ids.npy`` (int32 [n, k]), ``<prefix>scores.npy`` (fp32 [n, k]) and
        ``<prefix>users.npy`` (int64 [n], the user of each row) in out_dir, then commits them with ``manifest.json``; any
        earlier export in out_dir stops being readable when this one starts.  Device memory is bounded by the chunk: each chunk's
        lists go to the host through one of two pinned buffers while the next chunk is ranked.  Returns n."""
        ua = self._user_table(user_table)
        ids_np = self.check_users(users, ua.shape[0])
        _, ranks = _manifests(out_dir)
        return self._export(ua, ids_np, ids_np, out_dir, chunk, "", _new_export_id(), [MANIFEST] + list(ranks.values()))

    def _export(self, ua, ids_np: np.ndarray, names: np.ndarray, out_dir: str, chunk: int, prefix: str, export_id: int,
                stale, query: str = "users", meta=None) -> int:
        """export() of the rows ids_np of ua; ``users.npy`` gets `names` (the global ids of a row-sharded rank's local rows).
        query / meta: see _Files."""
        if chunk < 1:
            raise ValueError("chunk must be >= 1")
        n = ids_np.size
        files = _Files(out_dir, prefix, n, self.k, export_id, stale, query, meta)
        try:
            if n:
                files.arr[query][:] = names
                self._export_chunks(ua, ids_np, files.arr, chunk)
            files.commit()
        except BaseException:
            files.discard()
            raise
        return n

    def _export_chunks(self, ua, ids_np: np.ndarray, out, chunk: int) -> None:
        n, k, dev = ids_np.size, self.k, self.device
        c = min(chunk, n)
        pinned = dev.type == "cuda"
        host_users = torch.from_numpy(ids_np)
        if pinned:
            host_users = host_users.pin_memory()
        users_dev = torch.empty(c, dtype=torch.int64, device=dev)
        ids_dev = torch.empty(c, k, dtype=torch.int32, device=dev)
        sc_dev = torch.empty(c, k, dtype=torch.float32, device=dev)
        key_ws = self._key_ws(c)
        bufs = [(torch.empty(c, k, dtype=torch.int32, pin_memory=pinned), torch.empty(c, k, dtype=torch.float32, pin_memory=pinned))
                for _ in range(2)]
        done = [torch.cuda.Event() if pinned else None for _ in range(2)]
        pending = None                                 # (buffer index, first row, rows) of the chunk still on its way

        def drain(p):
            b, s, m = p
            if done[b] is not None:
                done[b].synchronize()
            out["ids"][s:s + m] = bufs[b][0][:m].numpy()
            out["scores"][s:s + m] = bufs[b][1][:m].numpy()

        for i, s in enumerate(range(0, n, c)):
            m, b = min(c, n - s), i % 2
            users_dev[:m].copy_(host_users[s:s + m], non_blocking=pinned)
            self._launch(ua, users_dev, m, ids_dev, sc_dev, k, key_ws)
            bufs[b][0][:m].copy_(ids_dev[:m], non_blocking=pinned)
            bufs[b][1][:m].copy_(sc_dev[:m], non_blocking=pinned)
            if done[b] is not None:
                done[b].record()
            if pending is not None:                    # the host writes the previous chunk while the device ranks this one
                drain(pending)
            pending = (b, s, m)
        drain(pending)


def _rank_prefix(rank: int, world: int) -> str:
    return f"rank{rank:05d}-of-{world:05d}."


def _new_export_id() -> int:
    return int.from_bytes(os.urandom(8), "little") >> 2


def _load_set(out_dir: str, prefix: str, meta: dict, query: str = "users"):
    arrs = {f: np.load(os.path.join(out_dir, f"{prefix}{f}.npy"), mmap_mode="r") for f in ("ids", "scores", query)}
    n, k = meta["n"], meta["k"]
    if arrs["ids"].shape != (n, k) or arrs["scores"].shape != (n, k) or arrs[query].shape != (n,):
        raise ValueError(f"{out_dir}: the {prefix}*.npy files do not have the shapes their manifest names")
    return arrs


# the readers of the export formats that share the file logic above: a directory of one kind is refused by the other's reader
READERS = {FORMAT: "recommendations (mmssl_b200.recommend.read)",
           "mmssl_b200.similar.v1": "similar items (mmssl_b200.similar.read)",
           "mmssl_b200.audience.v1": "audiences (mmssl_b200.audience.read)",
           "mmssl_b200.foldin.v1": "fold-in recommendations (mmssl_b200.foldin.read)"}


def _check_format(out_dir: str, meta: dict, fmt: str) -> None:
    got = meta.get("format", fmt)
    if got != fmt:
        raise ValueError(f"{out_dir}: holds an export of {READERS.get(got, repr(got))}, not of {READERS[fmt]}")


def read(out_dir: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(users [n] int64, ids [n, k] int32, scores [n, k] fp32) of the committed export in out_dir.  One-GPU layout (manifest.json):
    the files as written (memory-mapped), rows in the order the users were listed.  Row-sharded layout (rankRRRRR-of-WWWWW.json):
    every rank's rows, in ascending user order (the listed order among equal ids); every rank's manifest must be present and all
    must name the same export, so the files of an export that did not finish on every rank are never read as a whole.  A
    similar-items export (similar.py) is refused."""
    return _read(out_dir, "users", FORMAT, "recommendation")


def _read(out_dir: str, query: str, fmt: str, what: str):
    """read() of the exports whose row-id file is ``<query>.npy`` and whose manifests name format `fmt`."""
    one, ranks = _manifests(out_dir)
    if not one and not ranks:
        raise ValueError(f"{out_dir}: no committed {what} export (manifest.json or rankRRRRR-of-WWWWW.json)")
    if one and ranks:
        raise ValueError(f"{out_dir}: holds a one-GPU and a row-sharded export: remove one")
    if one:
        with open(os.path.join(out_dir, MANIFEST)) as fh:
            meta = json.load(fh)
        _check_format(out_dir, meta, fmt)
        arrs = _load_set(out_dir, "", meta, query)
        return arrs[query], arrs["ids"], arrs["scores"]
    worlds = sorted({w for _, w in ranks})
    if len(worlds) > 1:
        raise ValueError(f"{out_dir}: exports of several world sizes {worlds}: remove all but one")
    w = worlds[0]
    missing = [r for r in range(w) if (r, w) not in ranks]
    if missing:
        raise ValueError(f"{out_dir}: the export of world size {w} is incomplete: no {_manifest_name(_rank_prefix(missing[0], w))}")
    metas = []
    for r in range(w):
        with open(os.path.join(out_dir, ranks[(r, w)])) as fh:
            metas.append(json.load(fh))
        _check_format(out_dir, metas[-1], fmt)
    if len({m["export"] for m in metas}) != 1 or len({m["k"] for m in metas}) != 1:
        raise ValueError(f"{out_dir}: the rank files of world size {w} belong to different exports")
    parts = [_load_set(out_dir, _rank_prefix(r, w), metas[r], query) for r in range(w)]
    queries = np.concatenate([p[query] for p in parts])
    order = np.argsort(queries, kind="stable")
    return (queries[order], np.concatenate([p["ids"] for p in parts])[order],
            np.concatenate([p["scores"] for p in parts])[order])


def _sharded_stale(out_dir: str, rank: int, world: int):
    """The manifests a row-sharded export of (rank, world) removes before it writes: the rank's own, and on rank 0 those of a
    one-GPU export and of other world sizes."""
    stale = [_manifest_name(_rank_prefix(rank, world))]
    if rank == 0:
        _, ranks = _manifests(out_dir)
        stale += [MANIFEST] + [name for (_, w), name in ranks.items() if w != world]
    return stale


class ShardedRecommender:
    """``Recommender`` for a model whose tables are row-sharded over the ranks of a process group (rowshard_step.py): one per rank,
    holding only the exclusion rows of the rank's user block.  ``topk`` / ``export`` take the rank's padded [block, d] rows of
    the final user and item tables (``RowShardedHotStep.final_embeddings``) and the same list of global user ids on every rank;
    every rank all-gathers the item table once, then ranks the listed users of its block with local row ids against it (item
    ids stay global, so the tie rule is the one-GPU one).  A user's list depends only on its vector, the item table and its
    exclusion row, so every list is bitwise the one-GPU ``Recommender``'s on the gathered tables.  Nothing of the size of the
    lists travels between ranks: each rank returns and writes its own."""

    def __init__(self, exclude, part_u: RowPartition, part_i: RowPartition, rank: int, n_items: int, k: int, group=None,
                 device="cuda"):
        """exclude: (indptr [block + 1] rebased to 0, indices: global item ids sorted within each row) of the rank's user block."""
        if int(n_items) != part_i.n:
            raise ValueError(f"n_items {n_items} does not match the item partition ({part_i.n} rows)")
        if len(exclude[0]) != part_u.block + 1:
            raise ValueError(f"exclusion rows: indptr of {len(exclude[0])} entries, the user block needs {part_u.block + 1}")
        self.pu, self.pi, self.rank_id, self.group = part_u, part_i, int(rank), group
        self.n_users, self.n_items, self.k = part_u.n, int(n_items), int(k)
        if self.k < 1:
            raise ValueError("k must be >= 1")
        self.device = torch.device(device)
        self.exclude = _device_csr(exclude[0], exclude[1], self.device)

    @classmethod
    def from_shards(cls, sh, k: int, exclude: str = "train", group=None, device="cuda") -> "ShardedRecommender":
        """From ``dataset.ShardedDataset`` (rank and world as it was opened with): "train" = the pattern of the rank's ``ui`` rows,
        "seen" = their union with the ``val`` and ``test`` rows."""
        if exclude not in EXCLUDE:
            raise ValueError(f"exclude must be one of {EXCLUDE}, not {exclude!r}")
        pair = lambda b: (b.indptr, b.indices)
        rows = pair(sh.train_rows())
        if exclude == "seen":
            rows = union_csr(rows, pair(sh.held("val")), pair(sh.held("test")))
        return cls(rows, sh.part["user"], sh.part["item"], sh.rank, sh.n_items, k, group, device)

    @classmethod
    def from_rows(cls, train_items, test_set, val_set, n_users: int, n_items: int, part_u: RowPartition, part_i: RowPartition,
                  rank: int, k: int, exclude: str = "train", group=None, device="cuda") -> "ShardedRecommender":
        """From the reference's dicts; every rank keeps its block's exclusion rows."""
        if part_u.n != int(n_users):
            raise ValueError(f"n_users {n_users} does not match the user partition ({part_u.n} rows)")
        rows = _block_rows(exclusion_rows(train_items, test_set, val_set, exclude), part_u, rank)
        return cls(rows, part_u, part_i, rank, n_items, k, group, device)

    def check_users(self, users) -> np.ndarray:
        ids = _host_ids(users)
        if ids.size and (int(ids.min()) < 0 or int(ids.max()) >= self.n_users):
            raise ValueError(_BAD_USER)
        return ids

    def gather_items(self, i_local: torch.Tensor) -> torch.Tensor:
        """Collective.  [block, d] item rows of every rank -> the full [n_items, d] table."""
        return all_gather_rows(i_local.detach(), self.pi, self.group)

    def local(self, items: torch.Tensor) -> Recommender:
        """The one-GPU recommender of this rank's block against the gathered item table (user ids local to the block)."""
        return Recommender(items, self.exclude, self.k)

    def mine(self, ids: np.ndarray) -> np.ndarray:
        """Positions in `ids` of the users in this rank's block."""
        return np.nonzero(ids // self.pu.block == self.rank_id)[0]

    def topk(self, u_local: torch.Tensor, i_local: torch.Tensor, users):
        """Collective.  (ids [m, k] int64, scores [m, k] fp32, positions [m] host int64): the lists of the m listed users that are
        in this rank's block, and where they stand in `users`."""
        ids = self.check_users(users)
        rec = self.local(self.gather_items(i_local))
        pos = self.mine(ids)
        got_ids, got_sc = rec.topk(u_local, ids[pos] - self.rank_id * self.pu.block)
        return got_ids, got_sc, pos

    def export(self, u_local: torch.Tensor, i_local: torch.Tensor, users, out_dir: str, chunk: int = 1 << 16) -> int:
        """Collective (the export id and the item gather).  Writes ``rankRRRRR-of-WWWWW.{ids,scores,users}.npy`` with this rank's
        users only, in their listed order (``users.npy`` holds global ids), and commits them with ``rankRRRRR-of-WWWWW.json``
        naming an export id shared by all ranks.  Each rank first removes its own manifest, and rank 0 those of a one-GPU export
        and of other world sizes, so ``read`` sees the new export only once every rank has committed it.  Returns the number
        of rows written."""
        ids = self.check_users(users)
        prefix = _rank_prefix(self.rank_id, self.pu.world)
        stale = _sharded_stale(out_dir, self.rank_id, self.pu.world)
        export_id = self.export_id()
        rec = self.local(self.gather_items(i_local))
        mine = ids[self.mine(ids)]
        return rec._export(rec._user_table(u_local), mine - self.rank_id * self.pu.block, mine, out_dir, chunk, prefix, export_id,
                           stale)

    def export_id(self) -> int:
        """Collective.  A fresh random id, the same on every rank."""
        return shared_export_id(self.rank_id, self.pu.world, self.device, self.group)


def shared_export_id(rank: int, world: int, device, group=None) -> int:
    """Collective.  A fresh random id, the same on every rank: rank 0's draw (the only non-zero term of a sum)."""
    export_id = _new_export_id() if rank == 0 else 0
    if world > 1:
        t = torch.tensor([export_id], dtype=torch.int64, device=device)
        dist.all_reduce(t, group=group)
        export_id = int(t.item())
    return export_id
