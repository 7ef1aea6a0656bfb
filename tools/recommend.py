"""Export the top-k recommendations of every user of a trained model (mmssl_b200/recommend.py).

    python tools/recommend.py DATA --checkpoint run.ckpt --k 20 [--exclude train|seen] --out DIR [--chunk N]
        DATA: a dataset directory in the reference format (dataset.ReferenceDataset); run.ckpt: a ``Trainer.save`` file of a run on
        it.  Rebuilds the Trainer with the checkpoint's shape, loads it and writes DIR/{ids,scores,users}.npy + manifest.json.
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/recommend.py --sharded CKPT_DIR \\
        --shards SHARD_DIR --k 20 [--exclude train|seen] --out DIR
        CKPT_DIR: a row-sharded checkpoint (``RowShardedHotStep.save``, any world size); SHARD_DIR: ``dataset.write_shards`` output
        of its dataset.  Each rank loads its rows (resharded to N), runs the eval-mode forward and writes
        DIR/rankRRRRR-of-WWWWW.{ids,scores,users}.npy + .json for the users of its block.
    Neither checkpoint kind stores id_cat_rate / model_cat_rate, which shape the eval-mode forward: a run trained with other
    values than the defaults (0.36 / 0.55) needs --id-cat-rate / --model-cat-rate, in both modes.

    --audience [--items FILE]: in either mode, export the audiences of items instead -- the top-k users of each item
        (mmssl_b200/audience.py) -- as DIR/{ids,scores,items}.npy (or rankRRRRR-of-WWWWW.*, a rank writing the items of its item
        block): of every item, or of the int64 item ids in FILE (.npy).  --exclude drops the users who had the item in training
        ("train") or also in val / test ("seen"); --chunk then counts items.

    --fold-in FILE.npz: in either mode, export the top-k items of users given by item lists instead (mmssl_b200/foldin.py): FILE
        holds ``indptr`` / ``indices`` (int64, one row of item ids per query) and optionally ``users`` (int64, the id of a trained
        user, or -1 for a user the model never trained on).  Writes DIR/{ids,scores,queries}.npy, ``queries`` = each list's row
        number in FILE.  Row-sharded: a rank takes the queries of the users of its block plus its contiguous share of the
        new-user queries and writes rankRRRRR-of-WWWWW.*.  --exclude adds the training ("train") or also the val / test ("seen")
        items of a trained user to the query's own; --chunk then counts queries.

``recommend.read(DIR)`` returns (users, ids, scores) of either layout, ``audience.read(DIR)`` (items, ids, scores),
``foldin.read(DIR)`` (queries, ids, scores).  Prints one JSON line (rank 0)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from mmssl_b200 import audience, checkpoint, foldin, recommend  # noqa: E402


def _items(a, n_items: int) -> np.ndarray:
    return np.load(a.items).astype(np.int64).reshape(-1) if a.items else np.arange(n_items, dtype=np.int64)


def _fold_queries(path: str):
    """((indptr, indices), users) of a --fold-in file; users -1 where the file has none."""
    with np.load(path) as f:
        rows = (f["indptr"].astype(np.int64), f["indices"].astype(np.int64))
        n = rows[0].size - 1
        users = f["users"].astype(np.int64).reshape(-1) if "users" in f.files else np.full(n, -1, np.int64)
    if users.size != n:
        raise SystemExit(f"{path}: {users.size} users for {n} query rows")
    return rows, users


def load_trainer(a, dev):
    from mmssl_b200.dataset import ReferenceDataset
    from mmssl_b200.trainer import Trainer, TrainerArgs
    st = checkpoint.load(a.checkpoint, kinds=("trainer",))
    meta, tr = st["meta"], st["trainer"]
    d = int(meta["embed_size"])
    args = TrainerArgs(dataset=os.path.basename(os.path.normpath(a.data)), embed_size=d, batch_size=int(meta["batch_size"]),
                       head_num=int(meta["head_num"]), weight_size=str([d] * int(meta["n_layers"])), id_cat_rate=a.id_cat_rate,
                       model_cat_rate=a.model_cat_rate)
    if tr["sampler"] == "device":
        args.seed = int(tr["sampler_seed"])
    del st
    ds = ReferenceDataset.load(a.data)
    t = Trainer(ds, args, device=dev, sampler=tr["sampler"], log=None)
    t.load(a.checkpoint)
    return t


def one_gpu(a, dev):
    t = load_trainer(a, dev)
    if a.fold_in:
        rows, users = _fold_queries(a.fold_in)
        n = t.fold().export(rows, a.k, a.out, users, a.exclude, chunk=a.chunk)
        return dict(queries=n, users=t.n_users, items=t.n_items)
    if a.audience:
        aud, item_table = t.audience_ranker(a.k, a.exclude)         # what Trainer.audience ranks with
        n = aud.export(item_table, _items(a, t.n_items), a.out, chunk=a.chunk)
        return dict(audiences=n, users=t.n_users, items=t.n_items)
    rec, user_table = t.recommender(a.k, a.exclude)                 # what Trainer.recommend ranks with
    n = rec.export(user_table, np.arange(t.n_users, dtype=np.int64), a.out, chunk=a.chunk)
    return dict(users=n, items=t.n_items)


def load_sharded(a, dev, rank, world):
    """(the rank's ShardedDataset, its padded blocks of the final user and item tables) of the row-sharded checkpoint."""
    sh, step = load_sharded_step(a, dev, rank, world)
    u_f, i_f = step.final_embeddings()
    return sh, u_f, i_f


def load_sharded_step(a, dev, rank, world):
    """(the rank's ShardedDataset, its RowShardedHotStep with the checkpoint loaded)."""
    from mmssl_b200.dataset import ShardedDataset
    from mmssl_b200.engine import P_EI, P_EU
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
    st = checkpoint.read_sharded(a.sharded, world, rank)
    meta = st["meta"]
    sh = ShardedDataset.open(a.shards, rank, world)
    if (sh.n_users, sh.n_items) != (meta["n_users"], meta["n_items"]):
        raise SystemExit(f"{a.shards} holds {sh.n_users} x {sh.n_items}, the checkpoint {meta['n_users']} x {meta['n_items']}")
    # parameters of the right shapes (the load below overwrites every value): the replicated ones from the file, the two tables
    # as full-height placeholders that shard_problem_from_disk cuts into this rank's blocks
    P = {k: v for k, v in st["model"].items() if k not in (P_EU, P_EI)}
    P[P_EU] = torch.zeros(meta["n_users"], meta["embed_size"])
    P[P_EI] = torch.zeros(meta["n_items"], meta["embed_size"])
    Pl, fl, gl, pu, pi = shard_problem_from_disk(a.shards, P, rank, world, dev)
    B = int(meta["batch_size"])
    cfg = HotStepConfig(embed_size=int(meta["embed_size"]), n_layers=int(meta["n_layers"]), head_num=int(meta["head_num"]), batch_size=B,
                        id_cat_rate=a.id_cat_rate, model_cat_rate=a.model_cat_rate)
    step = RowShardedHotStep(Pl, fl, gl, cfg, B, pu, pi, rank)
    del st, P
    step.load(a.sharded)
    return sh, step


def fold_share(users: np.ndarray, part_u, rank: int) -> np.ndarray:
    """Row numbers of the --fold-in queries rank `rank` folds: those of the users of its block, then its contiguous share of the
    new-user (-1) queries, each in file order."""
    own = np.nonzero((users >= 0) & (users // part_u.block == rank))[0]
    new = np.nonzero(users < 0)[0]
    lo, hi = (new.size * rank) // part_u.world, (new.size * (rank + 1)) // part_u.world
    return np.concatenate([own, new[lo:hi]])


def sharded_fold_in(a, dev, rank, world):
    sh, step = load_sharded_step(a, dev, rank, world)
    rows, users = _fold_queries(a.fold_in)
    if users.size and int(users.max()) >= sh.n_users:
        raise SystemExit(f"{a.fold_in}: a user id outside [0, {sh.n_users})")
    fi = foldin.ShardedFoldIn.from_dataset(step.fold_tables(), sh, a.model_cat_rate)
    pick = fold_share(users, sh.part["user"], rank)
    n = fi.export(foldin.take_rows(rows, pick), a.k, a.out, users[pick], a.exclude, chunk=a.chunk, names=pick)
    return dict(queries=int(rows[0].size - 1), users=sh.n_users, items=sh.n_items, rows_written_by_rank0=n)


def sharded(a, dev, rank, world):
    if a.fold_in:
        return sharded_fold_in(a, dev, rank, world)
    sh, u_f, i_f = load_sharded(a, dev, rank, world)
    if a.audience:
        aud = audience.ShardedAudience.from_shards(sh, a.k, a.exclude, device=dev)
        n = aud.export(u_f, i_f, _items(a, sh.n_items), a.out, chunk=a.chunk)
        return dict(users=sh.n_users, items=sh.n_items, rows_written_by_rank0=n)
    rec = recommend.ShardedRecommender.from_shards(sh, a.k, a.exclude, device=dev)
    n = rec.export(u_f, i_f, np.arange(sh.n_users, dtype=np.int64), a.out, chunk=a.chunk)
    return dict(users=sh.n_users, items=sh.n_items, rows_written_by_rank0=n)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("data", nargs="?", help="dataset directory (reference format), with --checkpoint")
    ap.add_argument("--checkpoint", help="a Trainer.save file")
    ap.add_argument("--sharded", help="a row-sharded checkpoint directory (under torch.distributed.run)")
    ap.add_argument("--shards", help="dataset.write_shards output of the dataset, with --sharded")
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--exclude", choices=recommend.EXCLUDE, default="train")
    ap.add_argument("--out", required=True)
    ap.add_argument("--chunk", type=int, default=1 << 16, help="users (items with --audience) ranked per launch (bounds the device memory)")
    ap.add_argument("--audience", action="store_true", help="export the top-k users of items instead of the top-k items of users")
    ap.add_argument("--items", help="with --audience: a .npy of the item ids to rank (default: every item)")
    ap.add_argument("--fold-in", help="a .npz of query rows (indptr, indices, optional users): export their top-k items instead")
    # both rates shape the eval-mode forward and neither checkpoint kind stores them: give the trained run's values
    ap.add_argument("--id-cat-rate", type=float, default=0.36, help="the run's id_cat_rate (not in its checkpoint; default 0.36)")
    ap.add_argument("--model-cat-rate", type=float, default=0.55, help="the run's model_cat_rate (not in its checkpoint; default 0.55)")
    a = ap.parse_args(argv)
    if bool(a.sharded) == bool(a.checkpoint) or (a.sharded and not a.shards) or (a.checkpoint and not a.data):
        ap.error("give DATA --checkpoint FILE, or --sharded DIR --shards DIR")
    if a.items and not a.audience:
        ap.error("--items needs --audience")
    if a.fold_in and a.audience:
        ap.error("--fold-in and --audience are two different exports: give one")
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    t0 = time.perf_counter()
    if a.sharded:
        own = world > 1 and not dist.is_initialized()       # (a caller may have set up the process group already)
        if own:
            dist.init_process_group("nccl", device_id=dev)
        res = sharded(a, dev, rank, world)
        if world > 1:
            dist.barrier()
        if own:
            dist.destroy_process_group()
    else:
        res = one_gpu(a, dev)
    res.update(k=a.k, exclude=a.exclude, n_gpus=world, out=os.path.abspath(a.out), seconds=round(time.perf_counter() - t0, 2))
    if rank == 0:
        print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
