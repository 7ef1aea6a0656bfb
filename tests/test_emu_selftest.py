"""The cuemu fiber emulator (tests/cuemu) checked on kernels with known answers, and shown to catch the classes of
bugs it exists to catch: order-dependent results from a missing barrier, barrier deadlocks from wrong shuffle masks,
inline PTX it cannot run, invalid launch configurations."""
import ctypes as C

import numpy as np
import pytest

from tests.cuemu import harness


def _run(which, a=None, b=None, c=None, n=0, block=64, grid=1):
    lib = harness.emu_lib()
    lib.cuemu_st_run.restype = C.c_int
    lib.cuemu_st_error.restype = C.c_char_p
    p = lambda x: C.c_void_p(0 if x is None else x.ctypes.data)
    rc = lib.cuemu_st_run(which, p(a), p(b), p(c), n, block, grid)
    return rc, lib.cuemu_st_error().decode()


@pytest.mark.parametrize("order", ["fwd", "rev", "shuffle:3"])
def test_shuffles_and_ballot(order):
    harness.set_order(order)
    n = 96
    out = np.zeros((5, n), np.int32)
    rc, _ = _run(0, out, block=n)
    assert rc == 0
    t = np.arange(n)
    v = t * 3 + 1
    lane = t % 32
    assert np.array_equal(out[0], v[t ^ 5])
    src = np.where((lane % 16) + 3 < 16, t + 3, t)
    assert np.array_equal(out[1], v[src])
    src = np.where((lane % 8) - 2 >= 0, t - 2, t)
    assert np.array_equal(out[2], v[src])
    assert np.array_equal(out[3], v[(t & ~15) | 7])
    ballot = sum(1 << l for l in range(32) if l % 3 == 0)
    assert np.array_equal(out[4].astype(np.uint32), np.full(n, ballot, np.uint32))


@pytest.mark.parametrize("order", ["fwd", "rev", "shuffle:1"])
def test_group_masks_and_block_reduce(order):
    harness.set_order(order)
    out = np.zeros(64, np.float32)
    assert _run(1, out, block=64)[0] == 0
    want = np.repeat((np.arange(64) + 1).reshape(4, 16).sum(1), 16)
    assert np.array_equal(out, want.astype(np.float32))
    x = np.arange(5000, dtype=np.float32) % 7
    acc, flags = np.zeros(1, np.float32), np.zeros(4, np.int32)
    assert _run(2, x, acc, flags, n=5000, block=256, grid=3)[0] == 0
    assert acc[0] == x.sum() and flags.tolist() == [1, 1, 128, 1]


@pytest.mark.parametrize("limit", [64, 40, 17, 1])
def test_exited_threads_do_not_block(limit):
    harness.set_order("fwd")
    out = np.zeros(64, np.int32)
    assert _run(3, out, n=limit, block=64)[0] == 0
    want = np.zeros(64, np.int32)
    for w in range(2):
        live = max(0, min(32, limit - 32 * w))
        if live == 32:
            want[32 * w:32 * w + 32] = 32
    # partially exited warps: the values of exited lanes are undefined on the hardware; only full warps are compared
    full = [w for w in range(2) if limit >= 32 * (w + 1)]
    for w in full:
        assert np.array_equal(out[32 * w:32 * w + 32], want[32 * w:32 * w + 32])
    assert np.all(out[limit:] == 0)


def test_missing_barrier_is_order_dependent():
    res = []
    for order in ("fwd", "rev"):
        harness.set_order(order)
        out = np.zeros(64, np.int32)
        assert _run(4, out)[0] == 0
        res.append(out.copy())
    assert not np.array_equal(res[0], res[1])      # this is how a race shows up under the emulator


def test_deadlock_ptx_and_bad_configuration_are_reported():
    harness.set_order("fwd")
    out = np.zeros(64, np.int32)
    rc, msg = _run(6, out)
    assert rc != 0 and "deadlock" in msg and "st_bad_mask" in msg
    out[:] = 0
    rc, msg = _run(7, out)
    assert rc == 0 and out[0] == 1                  # griddepcontrol.wait is accepted
    out[1] = 7
    rc, msg = _run(7, out)
    assert rc != 0 and "multimem" in msg
    rc, msg = _run(8, np.zeros(5 * 2048, np.int32))
    assert rc != 0 and "invalid launch configuration" in msg
    assert _run(0, np.zeros((5, 32), np.int32), block=32)[0] == 0     # the error does not stick to later launches


def test_cache_hinted_loads_and_stores():
    """common.cuh's L1 / L2-hinted accesses (SpMM impl bits 7 and 8) are plain loads and stores in the model, both branches of
    the predicated hot / cold load included."""
    harness.set_order("fwd")
    a = np.arange(1, 25, dtype=np.float32)
    a.view(np.int32)[20] = 12345
    out = np.zeros(16, np.float32)
    rc, msg = _run(9, a, out)
    assert rc == 0, msg
    assert out[:10].tolist() == [1, 2, 7, 8, 9, 14, 19, 20, 12345, 22]
    assert out[12:].tolist() == [2, 3, 8, 9]
