"""Checkpoints of a training run: one ``torch.save`` dict per file, written atomically, read back into the live buffers.

Layout of a file (``FORMAT``):
  format   "mmssl_b200.ckpt.v1"
  kind     "hotstep" | "fullstep" | "trainer" | "rowshard"
  meta     the shape of the run a checkpoint belongs to (``META_FIELDS``): loading into another shape is refused by field name
  model    parameters under the reference's state_dict keys (Models.MMSSL; a Trainer file carries the whole module, unused
           registered parameters included, so ``MMSSL.load_state_dict(ckpt["model"])`` takes it as it is)
  optim    AdamW moments ``m`` / ``v`` of the seven live parameters and the step counter ``step``
  D, D_optim            (fullstep, trainer) ``Discriminator`` state_dict and its Adam moments / step
  fullstep              (fullstep, trainer) iteration in the epoch, collected top-k pairs, pairs the modality graphs were built from
  trainer               (trainer) epoch loop bookkeeping, sampler position, RNG states
  rows     (rowshard) the global row ranges [lo, hi) of the user / item table rows this file holds

A row-sharded run writes one file per rank into a generation directory that a manifest commits once every rank has written
(``save_sharded``); ``read_sharded`` reassembles the row blocks of any world size from the committed files that overlap them,
memory-mapped, so a run moves from N ranks to M, and M = 1 gives the state of a plain ``HotStep``."""
from __future__ import annotations

import os
import random
import re
import shutil
import tempfile
from typing import Dict, Tuple

import numpy as np
import torch

FORMAT = "mmssl_b200.ckpt.v1"
META_FIELDS = ("n_users", "n_items", "embed_size", "n_layers", "head_num", "batch_size", "feat_widths", "train_nnz", "train_hash",
               "sampler_seed")

_M64 = (1 << 64) - 1


# ------------------------------------------------------------------------------------------ training-matrix fingerprint
def _splitmix64(x: np.ndarray) -> np.ndarray:
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def pattern_hash(indptr, indices, n_cols: int, row0: int = 0) -> Tuple[int, int]:
    """(nnz, hash) of the sparsity pattern of a CSR block whose first row is global row ``row0``.  The hash is a sum over the
    edges (row, col) of a 64-bit mix of row * n_cols + col, so the hashes of row blocks add up to the hash of the whole matrix:
    a row-sharded run fingerprints the same matrix to the same value at any world size."""
    indptr = np.asarray(torch.as_tensor(indptr).cpu(), dtype=np.int64)
    indices = np.asarray(torch.as_tensor(indices).cpu(), dtype=np.int64)
    nnz = int(indptr[-1] - indptr[0]) if len(indptr) else 0
    rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.uint64) + np.uint64(row0), np.diff(indptr))
    with np.errstate(over="ignore"):
        key = rows * np.uint64(n_cols) + indices[indptr[0]:indptr[0] + nnz].astype(np.uint64)
        h = int(_splitmix64(key).sum(dtype=np.uint64)) if nnz else 0
    return nnz, h


def graph_fingerprint(g, row0: int = 0) -> Tuple[int, int]:
    """(nnz, hash) of the training pattern from the forward operand of the user-item graph (``graphs[0]``: the normalised
    training matrix, so its pattern is the matrix's)."""
    f = g.fwd
    return pattern_hash(f.rowptr, f.colidx[:f.nnz], f.n_cols, row0)


# ------------------------------------------------------------------------------------------ meta and validation
def make_meta(n_users, n_items, cfg, batch, feats, fingerprint) -> Dict[str, object]:
    return dict(n_users=int(n_users), n_items=int(n_items), embed_size=int(cfg.embed_size), n_layers=int(cfg.n_layers),
                head_num=int(cfg.head_num), batch_size=int(batch), feat_widths=[int(f.dim) for f in feats],
                train_nnz=int(fingerprint[0]), train_hash=int(fingerprint[1]))


def check_format(ckpt, kinds=None) -> None:
    if not isinstance(ckpt, dict) or ckpt.get("format") != FORMAT:
        got = ckpt.get("format") if isinstance(ckpt, dict) else type(ckpt).__name__
        raise ValueError(f"not a {FORMAT} checkpoint (format: {got!r})")
    if kinds is not None and ckpt.get("kind") not in kinds:
        raise ValueError(f"checkpoint kind {ckpt.get('kind')!r} cannot be loaded here (expected one of {tuple(kinds)})")


def check_meta(saved: Dict[str, object], have: Dict[str, object]) -> None:
    """Raises ``ValueError`` naming the first field in which the checkpoint's run differs from this one.  ``sampler_seed`` (a
    device sampler's seed) is compared when both runs have one."""
    for k in META_FIELDS:
        if k == "sampler_seed" and k not in saved:
            continue
        if k in have and saved.get(k) != have[k]:
            raise ValueError(f"checkpoint mismatch in {k}: saved {saved.get(k)!r}, this run {have[k]!r}")


def copy_into(dst: Dict[str, torch.Tensor], src: Dict[str, torch.Tensor], what: str) -> None:
    """In-place copy (the destination tensors are the static inputs of captured CUDA graphs: they keep their storage)."""
    for k, t in dst.items():
        if k not in src:
            raise ValueError(f"checkpoint has no {what} entry {k!r}")
        s = src[k]
        if tuple(s.shape) != tuple(t.shape):
            raise ValueError(f"checkpoint mismatch in {what} {k}: saved shape {tuple(s.shape)}, this run {tuple(t.shape)}")
    for k, t in dst.items():
        t.copy_(src[k])


# ------------------------------------------------------------------------------------------ RNG states
def rng_state(device) -> Dict[str, object]:
    """``random``, ``numpy.random``, torch CPU and (on a CUDA device) torch CUDA generator states -- what ``set_seed`` seeds."""
    np_state = np.random.get_state()
    st = dict(random=random.getstate(), numpy=(np_state[0], torch.from_numpy(np_state[1].astype(np.int64)), *np_state[2:]),
              torch=torch.get_rng_state())
    dev = torch.device(device)
    if dev.type == "cuda" and torch.cuda.is_available():
        st["cuda"] = torch.cuda.get_rng_state(dev)
    return st


def set_rng_state(st: Dict[str, object], device) -> None:
    random.setstate(st["random"])
    name, key, *rest = st["numpy"]
    np.random.set_state((name, np.asarray(key, dtype=np.int64).astype(np.uint32), *rest))
    torch.set_rng_state(st["torch"])
    dev = torch.device(device)
    if "cuda" in st and dev.type == "cuda" and torch.cuda.is_available():
        torch.cuda.set_rng_state(st["cuda"], dev)


# ------------------------------------------------------------------------------------------ files
def _host(obj):
    if isinstance(obj, torch.Tensor):
        return obj.detach().cpu()
    if isinstance(obj, dict):
        return {k: _host(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_host(v) for v in obj)
    return obj


def clone_state(obj):
    """Deep copy of a state dict on its device (a snapshot of the live buffers)."""
    if isinstance(obj, torch.Tensor):
        return obj.detach().clone()
    if isinstance(obj, dict):
        return {k: clone_state(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(clone_state(v) for v in obj)
    return obj


def save(ckpt: Dict[str, object], path: str) -> None:
    """Writes ``ckpt`` (device tensors are copied to the host) to a temporary file in the target's directory and renames it
    over ``path``: a write that is cut short leaves the previous checkpoint in place."""
    check_format(ckpt)
    path = os.path.abspath(path)
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(path) + ".", suffix=".tmp", dir=os.path.dirname(path))
    try:
        with os.fdopen(fd, "wb") as f:
            torch.save(_host(ckpt), f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise


def load(path: str, mmap: bool = False, kinds=None) -> Dict[str, object]:
    ckpt = torch.load(path, map_location="cpu", weights_only=True, mmap=mmap)
    check_format(ckpt, kinds)
    return ckpt


# ------------------------------------------------------------------------------------------ row-sharded runs
# A row-sharded checkpoint is a directory: one generation subdirectory per save (``step<S>-world<W>-<a|b>``, one file per rank)
# and MANIFEST.ckpt naming the complete generation.  Every rank writes its file into a fresh generation, all ranks meet at a
# barrier, then rank 0 replaces the manifest (atomically) and removes the other generations.  A pre-emption at any point
# leaves the manifest naming a generation whose files were all written, and all at the same step.
MANIFEST = "MANIFEST.ckpt"
_GENERATION = re.compile(r"step\d+-world\d+-[ab]")


def shard_file(directory: str, rank: int, world: int) -> str:
    return os.path.join(directory, f"rank{rank:05d}-of-{world:05d}.ckpt")


def read_manifest(directory: str) -> Dict[str, object]:
    path = os.path.join(directory, MANIFEST)
    if not os.path.exists(path):
        raise ValueError(f"{directory}: no committed row-sharded checkpoint ({MANIFEST} is missing)")
    return load(path, kinds=("rowshard-manifest",))


def committed_files(directory: str):
    """Paths of the files of the committed generation, in rank order."""
    man = read_manifest(directory)
    return [shard_file(os.path.join(directory, man["generation"]), r, man["world"]) for r in range(man["world"])]


def commit_sharded(directory: str, generation: str, world: int, step: int, meta: Dict[str, object]) -> None:
    """Rank 0, once every rank's file of ``generation`` is written: makes it the checkpoint, then drops the other generations."""
    save(dict(format=FORMAT, kind="rowshard-manifest", generation=generation, world=int(world), step=int(step), meta=meta),
         os.path.join(directory, MANIFEST))
    for name in os.listdir(directory):
        if name != generation and _GENERATION.fullmatch(name):
            shutil.rmtree(os.path.join(directory, name), ignore_errors=True)


def save_sharded(step, directory: str) -> None:
    """Collective over the ranks of a ``RowShardedHotStep``: each rank writes its file of a new generation, and rank 0 commits it
    after a barrier.  Saving at another world size into the same directory replaces the old files."""
    import torch.distributed as dist
    st = step.state_dict()                       # a collective too (the fingerprint)
    world, rank, n = step.pu.world, step.rank, int(st["optim"]["step"])
    os.makedirs(directory, exist_ok=True)
    current = read_manifest(directory)["generation"] if os.path.exists(os.path.join(directory, MANIFEST)) else None
    gen = f"step{n:010d}-world{world:05d}-a"
    if gen == current:                           # never overwrite the files of the committed generation
        gen = gen[:-1] + "b"
    os.makedirs(os.path.join(directory, gen), exist_ok=True)
    save(st, shard_file(os.path.join(directory, gen), rank, world))
    if world > 1:
        dist.barrier(group=step.group)           # every rank's file is on disk
    if rank == 0:
        commit_sharded(directory, gen, world, n, st["meta"])
    if world > 1:
        dist.barrier(group=step.group)           # no rank returns before the commit


def read_sharded(directory: str, world: int, rank: int) -> Dict[str, object]:
    """The state of rank ``rank`` of ``world`` from a row-sharded checkpoint written at any world size: the rank's padded row
    blocks of the two tables and of their moments (padding rows zero), assembled by global row id from the files whose rows
    overlap the block (memory-mapped: no rank reads the whole table), the replicated parameters from the first file.
    At world 1 the result is a ``HotStep`` checkpoint (kind "hotstep") of the whole tables."""
    from .engine import P_EI, P_EU
    from .parallel import RowPartition
    man = read_manifest(directory)
    w_saved, gdir = int(man["world"]), os.path.join(directory, man["generation"])

    def open_file(r: int) -> dict:
        path = shard_file(gdir, r, w_saved)
        f = load(path, mmap=True, kinds=("rowshard",))
        if int(f["optim"]["step"]) != int(man["step"]):
            raise ValueError(f"{path}: written at step {f['optim']['step']}, the checkpoint is at step {man['step']} "
                             "(files of different saves)")
        if f["meta"] != man["meta"]:
            raise ValueError(f"{path}: its meta differs from the checkpoint's (files of different runs)")
        return f
    first = open_file(0)
    meta = first["meta"]
    spaces = {P_EU: ("user", meta["n_users"]), P_EI: ("item", meta["n_items"])}
    files: Dict[int, dict] = {0: first}
    out = dict(format=FORMAT, kind="hotstep" if world == 1 else "rowshard", meta=dict(meta), model={},
               optim=dict(m={}, v={}, step=first["optim"]["step"]))
    for k, t in first["model"].items():
        if k not in spaces:
            out["model"][k] = t.clone()
            out["optim"]["m"][k] = first["optim"]["m"][k].clone()
            out["optim"]["v"][k] = first["optim"]["v"][k].clone()
    for k, (space, n) in spaces.items():
        part, saved = RowPartition(n, world), RowPartition(n, w_saved)
        lo, hi = part.bounds(rank)
        d = first["model"][k].shape[1]
        blocks = [torch.zeros(part.block, d, dtype=torch.float32) for _ in range(3)]
        for r in range(w_saved):
            slo, shi = saved.bounds(r)
            a, b = max(lo, slo), min(hi, shi)
            if a >= b:
                continue
            if r not in files:
                files[r] = open_file(r)
            f = files[r]
            if tuple(f["rows"][space]) != (slo, shi):
                raise ValueError(f"{shard_file(gdir, r, w_saved)}: holds {space} rows {tuple(f['rows'][space])}, expected {(slo, shi)}")
            for blk, src in zip(blocks, (f["model"][k], f["optim"]["m"][k], f["optim"]["v"][k])):
                blk[a - lo:b - lo] = src[a - slo:b - slo]
        out["model"][k], out["optim"]["m"][k], out["optim"]["v"][k] = blocks
    out["rows"] = {"user": RowPartition(meta["n_users"], world).bounds(rank), "item": RowPartition(meta["n_items"], world).bounds(rank)}
    return out
