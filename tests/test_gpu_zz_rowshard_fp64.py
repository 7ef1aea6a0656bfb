"""The row-sharded hot step (mmssl_b200/rowshard_step.py) against float64 on the H100, with the yardstick of
tests/rowshard_fp64.py (hotstep_fp64's measures and floors, the block-edge and rank-operand row classes, padding and
cross-rank equality exactly).

  a. world 1 in process: eight replays of the captured step drawing its batches with a ShardedTripleSampler, on both
     projection routes, each compared from the parameters the device held before it; one step at the Baby and the Sports shape
     with distinct modality graphs;
  b. worlds 2 and 3 (skipped where the GPUs are missing): ``python -m torch.distributed.run ... -m tests.rowshard_fp64`` with the
     nccl and the multicast exchange, both schedules, judged on rank 0; the multicast run also replays the captured step eight
     times and compares the replicated parameters across the ranks bitwise.

The emulator runs the same judge on gloo ranks at small sizes (tests/test_dist_emu_rowshard_fp64.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import hotstep_fp64 as H
from tests import rowshard_fp64 as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _eager(c):
    res = R.run_cases([c], 0, 1, "cuda")[0]
    R.judge(c, 1, {0: res}, what="world 1")


@pytest.mark.parametrize("route", ["tc/auto", "simt/simt"])
def test_captured_replays_with_sampler(route):
    """Capture (one warm-up optimiser step), then eight replays, each with new masks; the batch is the sampler's draw of the
    replay's step, read back from the step."""
    from mmssl_b200.dataset import CsrBlock
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.sampler import ShardedTripleSampler
    c = R.Case(U=1531, I=1237, d=64, B=257, modal="distinct", route=route, steps=8)
    p = R.case_problem(c)
    cfg = R.config(c)
    tr = p.train.tocsr()
    tr.sort_indices()
    pu = RowPartition(c.U, 1)
    smp = ShardedTripleSampler(CsrBlock(tr.indptr.astype(np.int64), tr.indices.astype(np.int32), None, tr.shape, 0, c.U), pu, 0,
                               seed=19)
    sh = R.shard_problem(p, cfg, 0, 1, "cuda", nce=route.split("/")[1], sampler=smp)
    sh.capture(warmup=1)
    gen = torch.Generator().manual_seed(43)
    recs, steps = [], []
    for _ in range(c.steps):
        masks = H.new_masks(c.I, c.d, c.drop, gen)
        for dst, m in zip(sh.masks, masks):
            dst.copy_(m)
        before = R.snapshot(sh)
        out5 = sh.replay().clone()
        torch.cuda.synchronize()
        rec = R.record(sh, out5, before)
        recs.append(rec)
        steps.append((*rec["idx"], masks))
    assert len({tuple(s[0][:8]) for s in steps}) == c.steps          # a fresh batch per replay
    recs.append(dict(schedule=sh.schedule))
    R.judge(c, 1, {0: recs}, what="captured, sampler", steps=steps, first_step=2)


@pytest.mark.parametrize("name", ["baby", "sports"])
def test_full_size_distinct_graphs(name):
    from mmssl_b200.synthetic import CONFIGS
    torch.set_num_threads(8)
    U, I, nnz, d, K, dv, dt = CONFIGS[name]
    for route in ("tc/auto", "simt/simt"):
        _eager(R.Case(U=U, I=I, d=d, K=K, B=1024, dv=dv, dt=dt, modal="distinct", route=route, seed=2022, train=name))


def _launch(world, exchange, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(port), "-m", "tests.rowshard_fp64", exchange]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    res = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert res["world"] == world and res["cases"] == 2 * len(R.gpu_cases(world)), res
    for route, tensor, measure, dev, f32 in res["ledger"]:          # into this process's ledger, by world and exchange
        H.LEDGER[(f"{route} w{world} {exchange}", tensor, measure)] = (dev, f32)
    if exchange == "multicast" and res["replays"] is None:
        pytest.skip("no NVSwitch multicast address: the captured step was not replayed")
    assert res["replays"] == (8 if exchange == "multicast" else 0), res


@pytest.mark.parametrize("exchange", ["nccl", "multicast"])
@pytest.mark.parametrize("world", [2, 3])
def test_multi_gpu(world, exchange):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _launch(world, exchange, 29550 + 2 * world + (exchange == "multicast"))


def test_zz_report_distances():
    """Largest distances to float64 seen by this module's tests, per route, tensor and measure (shown with -s)."""
    print("\n" + H.report())
