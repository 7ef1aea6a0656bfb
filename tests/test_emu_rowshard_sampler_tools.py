"""The exact integer exchange of the row-sharded sampler through NVSwitch multicast (mmssl_ids_to_limbs + mmssl_mc_allreduce_ids:
16-bit limbs summed by multimem.ld_reduce.add.v4.f32), played for several ranks in one process under the cuemu emulator, and
tools/config5_run.py
with --sampler device at toy size (one rank, eager steps)."""
import ctypes as C
import json
import runpy
import sys

import numpy as np
import pytest
import torch

from tests import test_emu_config5_tool as T5
from tests.cuemu import harness


@pytest.fixture
def emu(monkeypatch):
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    raw = harness.emu_lib()
    raw.cuemu_mc_clear()
    yield raw
    raw.cuemu_mc_clear()


@pytest.mark.parametrize("world", [2, 3])
def test_multicast_id_sum_is_exact(emu, world):
    """Every entry has one writing rank, zeros elsewhere: the sum is the written value, bitwise, also above 2^24 and 2^53 where an
    fp32 / fp64 sum of the values would round them, and for any 64-bit pattern."""
    from mmssl_b200 import _lib
    lib = _lib.load()
    n = 3 * 1000 + 5
    rng = np.random.default_rng(world)
    ids = torch.from_numpy(rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64))
    ids[:6] = torch.tensor([0, (1 << 24) + 1, (1 << 53) + 1, (1 << 62) + 3, -1, 65535])
    owner = torch.from_numpy(rng.integers(0, world, n))
    limbs = [torch.full((4 * n,), -7.0) for _ in range(world)]        # every rank's copy of the symmetric buffer
    for r in range(world):
        mine = torch.where(owner == r, ids, torch.zeros_like(ids))
        _lib.check(lib.mmssl_ids_to_limbs(_lib.ptr(mine), _lib.ptr(limbs[r]), n, None))
        assert bool(((limbs[r] >= 0) & (limbs[r] <= 65535) & (limbs[r] == limbs[r].round())).all())
    fake = torch.empty(4 * n * 4, dtype=torch.uint8)
    ptrs = (C.c_void_p * world)(*[t.data_ptr() for t in limbs])
    emu.cuemu_mc_register(C.c_uint64(fake.data_ptr()), C.c_uint64(4 * n * 4), world, ptrs)
    out = torch.full((n,), -1, dtype=torch.int64)
    _lib.check(lib.mmssl_mc_allreduce_ids(C.c_void_p(fake.data_ptr()), _lib.ptr(out), n, None))
    assert torch.equal(out, ids)


def test_multicast_id_sum_adds_every_rank(emu):
    """Several non-zero contributions per entry: the exact integer sum mod 2^64 (limb sums carry into the next limb)."""
    from mmssl_b200 import _lib
    lib = _lib.load()
    world, n = 3, 257
    rng = np.random.default_rng(9)
    vals = [torch.from_numpy(rng.integers(0, 1 << 62, n, dtype=np.int64)) for _ in range(world)]
    vals[0][0], vals[1][0], vals[2][0] = 0xFFFF, 0xFFFF, 0xFFFF                  # limb sums above 2^16 carry
    limbs = [torch.zeros(4 * n) for _ in range(world)]
    for r in range(world):
        _lib.check(lib.mmssl_ids_to_limbs(_lib.ptr(vals[r]), _lib.ptr(limbs[r]), n, None))
    fake = torch.empty(4 * n * 4, dtype=torch.uint8)
    emu.cuemu_mc_register(C.c_uint64(fake.data_ptr()), C.c_uint64(4 * n * 4), world, (C.c_void_p * world)(*[t.data_ptr() for t in limbs]))
    out = torch.zeros(n, dtype=torch.int64)
    _lib.check(lib.mmssl_mc_allreduce_ids(C.c_void_p(fake.data_ptr()), _lib.ptr(out), n, None))
    want = [sum(int(v[i]) for v in vals) % (1 << 64) for i in range(n)]
    assert [int(x) % (1 << 64) for x in out] == want


def test_config5_tool_with_device_sampler(monkeypatch, capsys):
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    real_gen = torch.Generator
    monkeypatch.setattr(torch, "Generator", lambda device=None: real_gen())
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(torch.cuda, "Event", T5._Event)
    monkeypatch.setattr(torch.cuda, "max_memory_allocated", lambda d=None: 0)
    monkeypatch.setattr(torch.cuda, "empty_cache", lambda: None)
    for k, v in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")):
        monkeypatch.setenv(k, v)
    monkeypatch.setattr(sys, "argv", ["config5_run.py", "--users", "300", "--items", "120", "--edges", "2500", "--embed-size", "64",
                                      "--dv", "64", "--dt", "64", "--steps", "1", "--batch", "64", "--no-graph", "--sampler", "device"])
    runpy.run_path(f"{T5.ROOT}/tools/config5_run.py", run_name="__main__")
    res = json.loads([l for l in capsys.readouterr().out.splitlines() if l.startswith("{")][-1])
    assert res["batches"] == "device sampler, fresh per step"
    assert all(np.isfinite(res["loss_first_step"]))
