"""Train with checkpoints and resume: the reference's epoch loop (mmssl_b200.trainer.Trainer) on a dataset directory in the
reference's format, writing a checkpoint after every epoch, or continuing from one.  Prints the save / load time and the
file size.

    python tools/resume_check.py DATA_DIR --epochs 3 --checkpoint run.ckpt                    # epochs 0..2, saved after each
    python tools/resume_check.py DATA_DIR --epochs 6 --resume run.ckpt --checkpoint run.ckpt  # continues at epoch 3

The shape flags (--batch, --embed, --sampler, --seed with the device sampler) must match the run that wrote the checkpoint: a
mismatch is refused by name.

    python tools/resume_check.py --config sports     # HotStep checkpoint of a synthetic bench.py shape: save / load time, size
"""
import argparse
import json
import os
import sys
from time import perf_counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("data", nargs="?", default="", help="dataset directory (train.json, val.json, test.json, train_mat, image_feat.npy, text_feat.npy)")
ap.add_argument("--epochs", type=int, default=3)
ap.add_argument("--checkpoint", default="", help="write the checkpoint here after every epoch")
ap.add_argument("--resume", default="", help="load this checkpoint before training")
ap.add_argument("--batch", type=int, default=1024)
ap.add_argument("--embed", type=int, default=64)
ap.add_argument("--sampler", default="reference", choices=["reference", "device"])
ap.add_argument("--seed", type=int, default=2022)
ap.add_argument("--cuda-graph", action="store_true")
ap.add_argument("--config", default="", help="instead of a dataset: time the HotStep checkpoint of this bench.py shape")
ap.add_argument("--dir", default="", help="with --config: where to write the file (default: a temporary directory)")
a = ap.parse_args()


def step_checkpoint(name: str) -> dict:
    """Save and load of one HotStep's checkpoint (parameters, AdamW moments, step) after one step, host <-> H100."""
    import tempfile
    import torch
    import bench
    from mmssl_b200 import checkpoint
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    ds, P, feats, graphs, _ = bench.build_problem(name, a.seed, "cuda")
    hs = HotStep(P, feats, graphs, HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=a.batch), batch=a.batch)
    hs.set_indices(*(torch.randint(0, n, (a.batch,)) for n in (ds.n_users, ds.n_items, ds.n_items)))
    hs.run()
    hs.meta()                                      # the fingerprint is computed once per step object: not part of the save
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory(dir=a.dir or None) as tmp:
        path = os.path.join(tmp, "hot.ckpt")
        t0 = perf_counter()
        checkpoint.save(hs.state_dict(), path)
        t_save = perf_counter() - t0
        t0 = perf_counter()
        hs.load_state_dict(checkpoint.load(path))
        torch.cuda.synchronize()
        t_load = perf_counter() - t0
        size = os.path.getsize(path)
    return dict(config=name, workload=f"{ds.n_users}x{ds.n_items}, d={ds.embed_size}", save_s=round(t_save, 3),
                load_s=round(t_load, 3), bytes=size)


if a.config:
    print(json.dumps(step_checkpoint(a.config)))
    sys.exit(0)
if not a.data:
    ap.error("a dataset directory or --config is needed")

import torch  # noqa: E402
from mmssl_b200.dataset import ReferenceDataset  # noqa: E402
from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed  # noqa: E402

args = TrainerArgs(dataset=os.path.basename(a.data.rstrip("/")), epoch=a.epochs, batch_size=a.batch, embed_size=a.embed,
                   weight_size=f"[{a.embed}, {a.embed}]", seed=a.seed, checkpoint=a.checkpoint)
set_seed(args.seed)
tr = Trainer(ReferenceDataset.load(a.data), args, sampler=a.sampler, cuda_graph=a.cuda_graph)
report = {}
if a.resume:
    torch.cuda.synchronize()
    t0 = perf_counter()
    tr.load(a.resume)
    torch.cuda.synchronize()
    report.update(load_s=round(perf_counter() - t0, 3), resumed_at_epoch=len(tr.history))
best, _ = tr.train()
report["best_recall"] = best
if a.checkpoint:
    torch.cuda.synchronize()
    t0 = perf_counter()
    tr.save(a.checkpoint)
    report.update(save_s=round(perf_counter() - t0, 3), bytes=os.path.getsize(a.checkpoint))
print(json.dumps(report))
