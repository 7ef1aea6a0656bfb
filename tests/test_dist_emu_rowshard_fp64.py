"""The row-sharded hot step (mmssl_b200/rowshard_step.py) against float64 on gloo ranks, every rank running the real kernel
sources under the cuemu emulator, with the yardstick of tests/rowshard_fp64.py: the losses, the table gradients assembled from
the ranks' blocks (norm-wise, row-wise, per class of rows including the block edges and the rows a rank's column-block operand
splits), the replicated gradients and each rank's AdamW update, for every optimiser step from the parameters the ranks held
before it; padding and cross-rank equality exactly.

The SpMM plan's cuts are lowered (8, 4, 32, 8) so that graphs of a few hundred rows have split and heavy rows.  Cases are
grouped: one spawn per world and group runs a list of them (start-up dominates a case)."""
import os
from dataclasses import replace

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import rowshard_fp64 as R
from tests.test_dist_emu import _MP, _free_port
from tests.test_gpu_zz_hotstep_fp64 import term_configs

CUTS = (8, 4, 32, 8)


def _worker(rank, world, port, cases, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        ret[rank] = R.run_cases(cases, rank, world, "cpu", cuts=CUTS)
    finally:
        dist.destroy_process_group()


def run_and_judge(cases, world):
    cases = [replace(c, cuts=CUTS) for c in cases]
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), cases, ret), nprocs=world, join=True)
    assert len(ret) == world
    res = {r: ret[r] for r in range(world)}
    for j, c in enumerate(cases):
        R.judge(c, world, {r: res[r][j] for r in range(world)}, what="emu")
    return res


def _terms(name, I=61, B=24):
    return tuple(term_configs(I, B)[name].items())


C = R.Case
# world 2: the six widths (every (G, C) instance of mmssl_reduce_rows_epilogue inside a whole step), K 1..3, 1 and 4 heads, the
# three modality-graph states, the three routes, both schedules
SHAPES = [
    C(d=32, K=1, heads=1, modal="distinct", route="simt/simt", schedule="reduce_scatter", kind="block edges"),
    C(d=64, K=3, heads=4, modal="alias", route="tc/auto", schedule="allgather", kind="block edges"),
    C(d=96, K=2, heads=1, modal="empty", route="simt/simt", schedule="reduce_scatter", kind="repeated"),
    C(d=128, K=1, heads=4, modal="distinct", route="simt/auto", schedule="reduce_scatter", kind="no edge"),
    C(d=192, K=3, heads=4, modal="alias", route="simt/simt", schedule="reduce_scatter", kind="one rank"),
    C(d=256, K=1, heads=1, modal="distinct", route="tc/auto", schedule="allgather", kind="plain"),
    C(d=64, K=2, heads=4, modal="distinct", route="tc/auto", schedule="reduce_scatter", kind="block edges"),
    # item 0 is heavy in the whole graph but only split in each rank's column block
    C(U=203, I=157, d=64, B=48, modal="distinct", route="simt/simt", schedule="reduce_scatter", kind="block edges", steps=2),
]
# each loss term dominant, both schedules
TERMS = [C(d=32, modal="distinct", schedule=s, kind="block edges", terms=_terms(t))
         for t in ("feat_reg dominant", "emb_reg dominant", "infonce dominant", "bpr only") for s in ("reduce_scatter", "allgather")]
# batches: B = 1, B larger than a block; no dropout (padded item rows of the projection hold the bias); four optimiser steps
BATCHES = [C(d=32, B=1, kind="plain", terms=_terms("bpr only")), C(d=32, B=48, U=61, I=43, kind="repeated"),
           C(d=32, drop=0.0, modal="distinct", kind="block edges", terms=_terms("feat_reg dominant")),
           C(d=64, modal="distinct", route="simt/auto", kind="block edges", steps=4),
           C(d=32, modal="empty", schedule="allgather", kind="one rank", steps=4)]


@pytest.mark.parametrize("group", ["shapes", "terms", "batches"])
def test_world_two(group):
    run_and_judge({"shapes": SHAPES, "terms": TERMS, "batches": BATCHES}[group], 2)


# world 3: uneven blocks; I = 4 leaves the third rank without any item row (block 2, rank 2 owns [4, 4))
WORLD3 = [C(d=32, modal="distinct", kind="block edges", steps=2),
          C(d=96, K=1, modal="alias", route="tc/auto", schedule="allgather", kind="one rank", steps=2),
          C(U=11, I=4, d=32, B=8, modal="distinct", kind="block edges", steps=4),
          C(U=11, I=4, d=64, B=8, modal="alias", schedule="allgather", kind="plain", steps=3, drop=0.0)]


def test_world_three():
    run_and_judge(WORLD3, 3)
