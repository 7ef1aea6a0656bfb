"""2-GPU test of the row-sharded propagation with the all-gather fused into the SpMM epilogue
(symmetric memory + multimem.st).  Skipped on single-GPU machines."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("mode", ["fused", "nccl"])
def test_row_sharded_chain_two_gpus(mode):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541" if mode == "fused" else "29542", os.path.join(ROOT, "tools", "rowshard_bench.py"), "tiktok", "check"]
    if mode == "fused":
        cmd.append("fused")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
    res = json.loads(line)
    assert res["n_gpus"] == 2 and res["max_rel_err_vs_1gpu"] < 1e-4
    if mode == "fused":
        assert res["exchange"].startswith("fused-in-SpMM")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_fused_dp_optimizer_two_gpus():
    """multimem reduce-scatter + sharded AdamW + multimem all-gather in one kernel == NCCL all-reduce(mean) + mmssl_adamw."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", os.path.join(ROOT, "tools", "dp_fused_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert res["n_gpus"] == 2 and res["max_rel_err_vs_nccl_path"] < 1e-6
