"""The two kernels that connect a batch of global row ids to a rank's row block [lo, hi) (csrc/shard.cu, used by the row-sharded
hot step): ``gather_owned`` must copy the owned rows bitwise and write +0 for every other id; ``scatter_add_owned`` must add
the owned rows' sources into a table that already holds values, duplicates included (a float4 atomicAdd per 16 bytes), within
the recursive-summation bound of the float64 sum, and leave every row it does not own -- and the padding beyond d of every
row -- bitwise untouched.  Widths 4 and the six library widths, leading dimensions larger than d, ids at lo - 1, lo, hi - 1, hi
and far out of range, lo == hi and n = 0.  The check_* bodies also run on the CPU under the cuemu emulator
(tests/test_emu_shard_kernels.py)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
WIDTHS = (4, 32, 64, 96, 128, 192, 256)
ROWS = 37


def _ids(lo, hi, n_table, gen, n=96):
    """Edge ids of [lo, hi) and of its neighbours, ids far out of range on both sides, then random ids in and around the block."""
    edge = [lo - 1, lo, hi - 1, hi, -1, -(1 << 40), n_table + 5, 1 << 40, 0, n_table - 1]
    rnd = torch.randint(max(lo - 3, 0), hi + 3, (n - len(edge),), generator=gen).tolist()
    return torch.tensor(edge + rnd, dtype=torch.int64)


def _block(d, ld, gen):
    """[ROWS, ld] storage with random values everywhere (the columns beyond d included); the kernel sees the [:, :d] view."""
    return torch.randn(ROWS, ld, generator=gen)


def check_gather_owned(d, lo, hi, n=96):
    from mmssl_b200.rowshard_step import gather_owned
    gen = torch.Generator().manual_seed(d * 1000 + lo * 10 + hi)
    ld, ldo = d + 4, d + 12
    n_table = hi + 20                       # global ids the batch may name
    tab = _block(d, ld, gen)[:max(hi - lo, 1)]
    idx = _ids(lo, hi, n_table, gen, n) if n else torch.zeros(0, dtype=torch.int64)
    out_store = torch.full((max(n, 1), ldo), float("nan"))
    dev_tab, dev_idx, dev_out = tab.cuda(), idx.cuda(), out_store.cuda()
    gather_owned(dev_tab[:, :d], dev_idx, lo, hi, dev_out[:n, :d])
    torch.cuda.synchronize()
    got = dev_out.cpu()
    assert torch.isnan(got[:, d:]).all(), "gather_owned wrote past d"
    if n == 0:
        assert torch.isnan(got).all()
        return
    ids = idx.numpy()
    own = (ids >= lo) & (ids < hi)
    want = torch.zeros(n, d)
    want[torch.from_numpy(own)] = tab[torch.from_numpy(ids[own] - lo), :d]
    g = got[:n, :d]
    assert np.array_equal(g.numpy().view(np.uint32), want.numpy().view(np.uint32)), \
        f"d={d} [{lo}, {hi}): rows differ at {np.nonzero((g != want).any(1).numpy())[0].tolist()}"   # +0, not -0, for the others


def check_scatter_add_owned(d, lo, hi, n=96, dup=64):
    """`dup` copies of one owned id (hi - 1) first, then edge and random ids; sources of mixed sign and magnitude."""
    from mmssl_b200.rowshard_step import scatter_add_owned
    gen = torch.Generator().manual_seed(d * 1000 + lo * 10 + hi + 7)
    ld, lds = d + 4, d + 8
    n_table = hi + 20
    tab = _block(d, ld, gen)[:max(hi - lo, 1)]
    idx = torch.zeros(0, dtype=torch.int64)
    if n:
        hot = torch.full((dup,), hi - 1 if hi > lo else lo, dtype=torch.int64)
        idx = torch.cat([hot, _ids(lo, hi, n_table, gen, n)])
    m = idx.numel()
    src = torch.randn(max(m, 1), lds, generator=gen) * torch.exp(torch.randn(max(m, 1), 1, generator=gen) * 3)
    dev_tab, dev_idx, dev_src = tab.cuda(), idx.cuda(), src.cuda()
    scatter_add_owned(dev_tab[:, :d], dev_idx, lo, hi, dev_src[:m, :d])
    torch.cuda.synchronize()
    got = dev_tab.cpu()
    assert np.array_equal(got[:, d:].numpy().view(np.uint32), tab[:, d:].numpy().view(np.uint32)), "scatter_add_owned wrote past d"
    ids = idx.numpy()
    own = (ids >= lo) & (ids < hi)
    touched = np.zeros(tab.shape[0], bool)
    touched[ids[own] - lo] = True
    untouched = torch.from_numpy(~touched)
    assert np.array_equal(got[untouched].numpy().view(np.uint32), tab[untouched].numpy().view(np.uint32)), \
        f"d={d} [{lo}, {hi}): rows without an owned id changed"
    if hi == lo or m == 0:
        return
    # float64 sum and the recursive-summation bound gamma_(k-1) sum|terms| = (k - 1) u / (1 - (k - 1) u) sum|terms|, u = 2^-24, of
    # the k terms of each element (table value + sources), whatever order the atomics land in
    s64 = tab[:, :d].double().clone()
    mag = tab[:, :d].double().abs()
    cnt = np.ones(tab.shape[0], np.int64)
    for j in np.nonzero(own)[0]:
        r = ids[j] - lo
        s64[r] += src[j, :d].double()
        mag[r] += src[j, :d].double().abs()
        cnt[r] += 1
    ku = torch.from_numpy(cnt - 1).double()[:, None] * 2.0 ** -24
    bound = ku / (1 - ku) * mag
    err = (got[:, :d].double() - s64).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"d={d} [{lo}, {hi}): {int(bad.sum())} elements beyond the summation bound, worst "
                                 f"{float((err - bound).max()):.3g} over it; terms in the hot row {int(cnt[hi - 1 - lo])}")
    assert int(cnt[hi - 1 - lo]) >= dup + 1


# (lo, hi): a middle block, the first block, lo == hi, a one-row block
BLOCKS = ((20, 37), (0, 17), (9, 9), (30, 31))


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("lo,hi", BLOCKS)
def test_gather_owned(d, lo, hi):
    check_gather_owned(d, lo, hi)


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("lo,hi", BLOCKS)
def test_scatter_add_owned(d, lo, hi):
    check_scatter_add_owned(d, lo, hi)


@pytest.mark.parametrize("d", [4, 96])
def test_empty_batch(d):
    check_gather_owned(d, 20, 37, n=0)
    check_scatter_add_owned(d, 20, 37, n=0)
