"""The row-sharded device sampler on the GPU (sampler.ShardedTripleSampler): at world 1 both paths bitwise DeviceTripleSampler at
Baby and 1M users; the captured RowShardedHotStep with the sampler draws DeviceTripleSampler's batch of each replay's step and
agrees with HotStep on it; on 2 GPUs (skipped below 2) tools/rowshard_sampler_bench.py `check` reports bitwise batches on every
rank, through NCCL and the multicast exchange."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
TOL = 1e-4                  # the row-sharded step against HotStep on one GPU (tests/test_gpu_zz_dist_step.py)


def _tool():
    spec = importlib.util.spec_from_file_location("rowshard_sampler_bench", os.path.join(ROOT, "tools", "rowshard_sampler_bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("name", ["baby", "syn1m"])
def test_world_one_bitwise(name):
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.sampler import DeviceTripleSampler, ShardedTripleSampler
    T = _tool()
    U, I = T.SIZES[name]
    rows = T.device_rows(U, I, 0, U, 3, "cuda")
    full = DeviceTripleSampler(T.to_scipy(rows), seed=5)
    mine = ShardedTripleSampler(rows, RowPartition(U, 1), 0, seed=5)
    n = full.exist.numel()
    assert mine.n_exist == n
    for b in (1, 777, 1024, 1025, 4096, 16384, n, n + 1):
        for step in (0, 3):
            want = full.sample_into(torch.zeros(3, b, dtype=torch.int64, device="cuda"), step=step)
            got = mine.sample_into(torch.full((3, b), -1, dtype=torch.int64, device="cuda"), step=step)
            assert torch.equal(got, want), (b, step)


@pytest.mark.parametrize("batch", [1024, 4096])
def test_captured_rowshard_step_draws_each_replays_batch(batch):
    """World 1, Tiktok: N replays of the captured step with the sampler.  The step counter is set before each replay (no
    optimiser step, so the parameters stay put): the replay's batch is DeviceTripleSampler's at that step, bitwise, and its
    losses and gradients are HotStep's on the same batch within the row-sharded tolerance."""
    import bench
    from mmssl_b200.dataset import CsrBlock
    from mmssl_b200.engine import LIVE, P_EI, P_EU
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem
    from mmssl_b200.sampler import DeviceTripleSampler, ShardedTripleSampler
    from tests.golden_util import rel_err
    ds, P_cpu, feats_cpu, _, _ = bench.build_problem("tiktok", 2022, None)
    _, Pd, feats, graphs, _ = bench.build_problem("tiktok", 2022, "cuda")
    cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=batch)
    Pl, fl, gl, pu, pi = shard_problem(P_cpu, feats_cpu, ds.ui_norm, ds.iu_norm, 0, 1, "cuda")
    R = ds.train.tocsr()
    R.sort_indices()
    import numpy as np
    smp = ShardedTripleSampler(CsrBlock(R.indptr.astype(np.int64), R.indices.astype(np.int32), None, R.shape, 0, R.shape[0]), pu, 0,
                               seed=13)
    sh = RowShardedHotStep(Pl, fl, gl, cfg, batch, pu, pi, 0, optimizer_step=False, sampler=smp)
    hs = HotStep(Pd, feats, graphs, cfg, batch=batch, optimizer_step=False, sampler=DeviceTripleSampler(R, seed=13))
    g = torch.Generator().manual_seed(7)
    masks = tuple(((torch.rand(ds.n_items, ds.embed_size, generator=g) >= cfg.drop_rate) / (1 - cfg.drop_rate)).float().cuda()
                  for _ in range(2))
    hs.masks, sh.masks = masks, masks
    sh.capture()
    ref = DeviceTripleSampler(R, seed=13)
    seen = set()
    for n in (0, 1, 2, 7):
        sh.step_dev.fill_(n)
        hs.step_dev.fill_(n)
        out = sh.replay().clone()
        want_idx = ref.sample_into(torch.zeros(3, batch, dtype=torch.int64, device="cuda"), step=n)
        assert torch.equal(sh.idx, want_idx), n
        seen.add(tuple(sh.idx[0, :8].tolist()))
        want = hs.run().clone()
        assert torch.equal(hs.idx, sh.idx), n
        assert float(((out - want).abs() / want.abs().clamp_min(1e-12)).max()) < TOL, n
        for k in LIVE:
            got_g = sh.grads[k][:pu.n] if k == P_EU else sh.grads[k][:pi.n] if k == P_EI else sh.grads[k]
            assert rel_err(got_g, hs.grads[k]) < TOL, (n, k)
    assert len(seen) == 4                              # a fresh batch per replay
    assert sh.meta()["sampler_seed"] == 13


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_sampler_two_gpus():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29547", os.path.join(ROOT, "tools", "rowshard_sampler_bench.py"), "check"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert res["n_gpus"] == 2 and res["check"] is True and res["comparisons"] > 0, res
