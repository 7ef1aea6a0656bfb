"""2-GPU test of the row-sharded WHOLE hot step (sorts last; skipped on single-GPU machines)."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("exchange", ["nccl", "mc"])
def test_row_sharded_whole_step_two_gpus(exchange):
    """rowshard_step.RowShardedHotStep on 2 GPUs == the single-GPU fused HotStep: the five loss terms and every live gradient of
    two steps, 1e-4 (the contract).  The same class is checked with 2 gloo ranks under the CPU emulator in tests/test_dist_emu.py;
    bench.py --gpus N repeats the check at sports / syn1m scale on every multi-GPU run (`row_shard.*.parity_vs_1gpu`)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29544" if exchange == "nccl" else "29545", os.path.join(ROOT, "tools", "rowshard_step_bench.py"), "tiktok", "check",
           "--steps", "5"] + (["mc"] if exchange == "mc" else [])
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert res["n_gpus"] == 2 and res["max_rel_err_vs_1gpu"] < 1e-4 and res["gathers_per_step"] > 0
    assert res["exchange"].startswith("NCCL") == (exchange == "nccl")
