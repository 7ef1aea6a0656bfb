"""Export the top-k similar items of every catalogue item of a trained model, or of new items given by their features
(mmssl_b200/similar.py).

    python tools/similar_items.py DATA --checkpoint run.ckpt --k 20 [--space model|image|text] --out DIR [--chunk N]
                                  [--features IMG.npy TXT.npy]
        DATA: a dataset directory in the reference format (dataset.ReferenceDataset); run.ckpt: a ``Trainer.save`` file of a run on
        it.  Rebuilds the Trainer with the checkpoint's shape, loads it and writes DIR/{ids,scores,items}.npy + manifest.json:
        every catalogue item's list, or with --features (space image or text) the lists of the rows of IMG.npy [m, Dv] /
        TXT.npy [m, Dt] against the whole catalogue (items.npy then holds the row numbers).
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/similar_items.py --sharded CKPT_DIR \\
        --shards SHARD_DIR --k 20 [--space model|image|text] --out DIR
        CKPT_DIR: a row-sharded checkpoint (``RowShardedHotStep.save``, any world size); SHARD_DIR: ``dataset.write_shards`` output
        of its dataset.  Each rank loads its rows (resharded to N), computes its block of the space's table and writes
        DIR/rankRRRRR-of-WWWWW.{ids,scores,items}.npy + .json for the items of its block.
    Neither checkpoint kind stores id_cat_rate / model_cat_rate, which shape the "model" space's eval-mode forward: a run trained
    with other values than the defaults (0.36 / 0.55) needs --id-cat-rate / --model-cat-rate, in both modes.

``similar.read(DIR)`` returns (items, ids, scores) of either layout.  Prints one JSON line (rank 0)."""
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

from mmssl_b200 import checkpoint, similar  # noqa: E402


def one_gpu(a, dev):
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
    sim = t.similar(a.k, a.space)                                  # what Trainer.similar_items ranks with
    if a.features:
        n = sim.export_features(np.load(a.features[0]), np.load(a.features[1]), a.out, chunk=a.chunk)
    else:
        n = sim.export(np.arange(t.n_items, dtype=np.int64), a.out, chunk=a.chunk)
    return dict(queries=n, items=t.n_items)


def sharded(a, dev, rank, world):
    from mmssl_b200.dataset import ShardedDataset
    from mmssl_b200.engine import P_EI, P_EU
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
    st = checkpoint.read_sharded(a.sharded, world, rank)
    meta = st["meta"]
    sh = ShardedDataset.open(a.shards, rank, world)
    if (sh.n_users, sh.n_items) != (meta["n_users"], meta["n_items"]):
        raise SystemExit(f"{a.shards} holds {sh.n_users} x {sh.n_items}, the checkpoint {meta['n_users']} x {meta['n_items']}")
    # parameters of the right shapes (the load below overwrites every value), as tools/recommend.py builds them
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
    if a.space == "model":
        table = step.final_embeddings()[1]
    else:
        table = step.projections()[0 if a.space == "image" else 1]
    sim = similar.ShardedSimilarItems(pi, rank, a.k, a.space, device=dev)
    n = sim.export(table, np.arange(sh.n_items, dtype=np.int64), a.out, chunk=a.chunk)
    return dict(queries=sh.n_items, items=sh.n_items, rows_written_by_rank0=n)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("data", nargs="?", help="dataset directory (reference format), with --checkpoint")
    ap.add_argument("--checkpoint", help="a Trainer.save file")
    ap.add_argument("--sharded", help="a row-sharded checkpoint directory (under torch.distributed.run)")
    ap.add_argument("--shards", help="dataset.write_shards output of the dataset, with --sharded")
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--space", choices=similar.SPACES, default="model")
    ap.add_argument("--features", nargs=2, metavar=("IMG.npy", "TXT.npy"),
                    help="feature rows of new items (with --checkpoint and --space image or text)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--chunk", type=int, default=1 << 16, help="items ranked per launch (bounds the device memory)")
    # both rates shape the eval-mode forward and neither checkpoint kind stores them: give the trained run's values
    ap.add_argument("--id-cat-rate", type=float, default=0.36, help="the run's id_cat_rate (not in its checkpoint; default 0.36)")
    ap.add_argument("--model-cat-rate", type=float, default=0.55, help="the run's model_cat_rate (not in its checkpoint; default 0.55)")
    a = ap.parse_args(argv)
    if bool(a.sharded) == bool(a.checkpoint) or (a.sharded and not a.shards) or (a.checkpoint and not a.data):
        ap.error("give DATA --checkpoint FILE, or --sharded DIR --shards DIR")
    if a.features and (a.sharded or a.space == "model"):
        ap.error("--features needs --checkpoint and --space image or text")
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
    res.update(k=a.k, space=a.space, features=bool(a.features), n_gpus=world, out=os.path.abspath(a.out),
               seconds=round(time.perf_counter() - t0, 2))
    if rank == 0:
        print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
