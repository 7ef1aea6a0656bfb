"""The device triple sampler (csrc/sampler.cu) bit for bit against its exact model (tests/sampler_model.py): the one-CTA claim
path at every batch size close to n_exist (where the claim rounds leave threads to the claim finish), the radix-select path at
every size class, rows that force the negative's complement fallback, item counts near 2^31, extreme seeds and steps from the
host and from the device counter, the row-sharded (owned) entry points block by block, and ShardedTripleSampler at world 1.
Also: the claim table is left clean, a user whose row holds every item is refused, and the distribution of users, positives
and negatives on the device.  The check_* bodies also run in the emulator at small sizes (tests/test_emu_sampler_exact.py)."""
import math

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests import sampler_model as S

PAIRS = [(0, 0), (2022, 1), (2 ** 63 + 5, 2 ** 31 - 1), (2 ** 64 - 1, 1)]      # (seed, step)
PAIRS_SHORT = [(2022, 0), (2 ** 64 - 1, 2 ** 31 - 1)]


def csr_of(row_lists, n_items):
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in row_lists])]).astype(np.int64)
    indices = np.concatenate([np.sort(np.asarray(r, np.int64)) for r in row_lists] + [np.zeros(0, np.int64)])
    return sp.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(len(row_lists), n_items))


def sparse_csr(n_exist, n_items=64, seed=0, empty_every=5):
    """n_exist users with 1..4 items, an empty row after every `empty_every`-th of them."""
    rng = np.random.default_rng(seed)
    rows = []
    for u in range(n_exist):
        rows.append(rng.choice(n_items, size=int(rng.integers(1, min(4, n_items) + 1)), replace=False).tolist())
        if u % empty_every == empty_every - 1:
            rows.append([])
    return csr_of(rows, n_items)


def edge_csr():
    """Rows that take the complement fallback (50 000 items, one or three missing at 0, n - 1 and mid-row), rows of degree 1,
    empty rows between them."""
    n = 50_000
    full = np.arange(n)
    rows = [np.delete(full, [0]), [], np.delete(full, [n - 1]), [7], np.delete(full, [n // 2]), [],
            np.delete(full, [0, n // 2, n - 1]), [49_999], [0], [], np.delete(full, [1, 2, n - 2])]
    return csr_of([np.asarray(r) for r in rows], n)


def dense40_csr():
    """40 items: rows of degree 39 (missing 0, 5 or 39) and 37, rows of degree 1, empty rows."""
    a = np.arange(40)
    rows = [np.delete(a, [5]), [], np.delete(a, [0, 20, 39]), [39], np.delete(a, [0]), [0], [], np.delete(a, [39]), [17]]
    return csr_of([np.asarray(r) for r in rows], 40)


def huge_items_csr(n_exist=300, seed=1):
    """n_items = 2^31 - 1: sparse rows whose ids reach the top of the range."""
    n_items = 2 ** 31 - 1
    rng = np.random.default_rng(seed)
    rows = [np.unique(np.concatenate([rng.integers(0, n_items, 3), [n_items - 1 - u % 2]])).tolist() for u in range(n_exist)]
    rows[5:5] = [[]]
    return csr_of(rows, n_items)


def one_cta(smp, b, seed, step, step_dev=False):
    out = torch.full((3, b), -1, dtype=torch.int64, device="cuda")
    smp.seed = seed
    if step_dev:
        smp.sample_into(out, step_dev=torch.full((1,), step, dtype=torch.int32, device="cuda"))
    else:
        smp.sample_into(out, step=step)
    return out.cpu().numpy()


def multi_direct(smp, b, seed, step, step_dev=False):
    from mmssl_b200 import _lib
    from mmssl_b200._lib import ptr, stream
    lib = _lib.load(require_device=True)
    n_exist = smp.exist.numel()
    nbytes = lib.mmssl_sampler_workspace_bytes(n_exist, b)
    ws = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    out = torch.full((3, b), -1, dtype=torch.int64, device="cuda")
    sd = torch.full((1,), step, dtype=torch.int32, device="cuda") if step_dev else None
    _lib.check(lib.mmssl_sample_triples_multi(ptr(smp.indptr), ptr(smp.indices), ptr(smp.exist), n_exist, smp.n_items, b, seed, ptr(sd),
                                              0 if step_dev else step, ptr(ws), ws.numel(), ptr(out[0]), ptr(out[1]), ptr(out[2]), stream()))
    return out.cpu().numpy()


def claim_clean(smp):
    return bool((smp.claim == 0x7FFFFFFF).all())


def check_one_cta(csr, batches, pairs, step_dev_too=True):
    """sample_into at batches <= 1024 bitwise the model; returns the number of threads the claim finish served and of triples that
    took the complement fallback."""
    from mmssl_b200.sampler import DeviceTripleSampler
    smp = DeviceTripleSampler(csr)
    rows = S.Rows(csr)
    fin = fb = 0
    for b in batches:
        assert b <= S.ONE_CTA_MAX
        for k, (seed, step) in enumerate(pairs):
            want, info = S.one_cta(rows, b, seed, step)
            got = one_cta(smp, b, seed, step, step_dev=step_dev_too and k == len(pairs) - 1)
            assert np.array_equal(got, want), (b, rows.n_exist, seed, step, (got != want).sum(axis=1))
            if b <= rows.n_exist:
                assert len(np.unique(got[0])) == b
            fin += info["finish"]
            fb += info["fallback"]
            assert claim_clean(smp), (b, seed, step)
    return fin, fb


def check_multi(csr, batches, pairs, step_dev_too=True):
    """The direct multi-CTA entry bitwise the model's select; sample_into too above 1024 triples."""
    from mmssl_b200.sampler import DeviceTripleSampler
    smp = DeviceTripleSampler(csr)
    rows = S.Rows(csr)
    fb = 0
    for b in batches:
        for k, (seed, step) in enumerate(pairs):
            want, info = S.multi(rows, b, seed, step)
            got = multi_direct(smp, b, seed, step, step_dev=step_dev_too and k == len(pairs) - 1)
            assert np.array_equal(got, want), (b, rows.n_exist, seed, step, (got != want).sum(axis=1))
            if b > S.ONE_CTA_MAX:
                assert np.array_equal(one_cta(smp, b, seed, step), want), (b, seed, step)
            fb += info["fallback"]
    return fb


def block_arrays(csr, lo, hi):
    """The rows [lo, hi) as the owned entry points take them: rebased indptr, int32 global item ids, local non-empty rows, and
    the block's first slot."""
    ip = csr.indptr.astype(np.int64)
    indptr = ip[lo:hi + 1] - ip[lo]
    indices = csr.indices[ip[lo]:ip[hi]].astype(np.int32)
    deg = np.diff(ip)
    exist = np.nonzero(deg[lo:hi] > 0)[0].astype(np.int64)
    return indptr, indices, exist, int((deg[:lo] > 0).sum())


def owned_call(csr, lo, hi, b, seed, step):
    from mmssl_b200 import _lib
    from mmssl_b200._lib import ptr, stream
    lib = _lib.load(require_device=True)
    indptr, indices, exist, slot_lo = block_arrays(csr, lo, hi)
    dev = lambda a: torch.from_numpy(a).to("cuda")
    indptr, indices, exist_t = dev(indptr), dev(indices), dev(exist) if len(exist) else torch.zeros(1, dtype=torch.int64, device="cuda")
    n_exist = int((np.diff(csr.indptr) > 0).sum())
    out = torch.full((3, b), -1, dtype=torch.int64, device="cuda")
    args = (ptr(indptr), ptr(indices), ptr(exist_t), slot_lo, slot_lo + len(exist), lo, n_exist, csr.shape[1], b, seed, None, step)
    if b <= S.ONE_CTA_MAX:
        claim = torch.empty(n_exist, dtype=torch.int32, device="cuda")
        _lib.check(lib.mmssl_sampler_init(ptr(claim), n_exist, stream()))
        _lib.check(lib.mmssl_sample_triples_owned(*args, ptr(claim), ptr(out[0]), ptr(out[1]), ptr(out[2]), stream()))
        assert bool((claim == 0x7FFFFFFF).all())
    else:
        nbytes = lib.mmssl_sampler_workspace_bytes(n_exist, b)
        ws = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda")
        _lib.check(lib.mmssl_sample_triples_multi_owned(*args, ptr(ws), ws.numel(), ptr(out[0]), ptr(out[1]), ptr(out[2]), stream()))
    return out.cpu().numpy(), slot_lo, slot_lo + len(exist)


def check_owned_blocks(csr, batches, worlds, pairs):
    """Each block of a 2- and 3-way row partition through the owned entry points: the model's batch with zeros outside the
    block's slots, and the blocks sum to the one-GPU batch."""
    from mmssl_b200.parallel import RowPartition
    rows = S.Rows(csr)
    for world in worlds:
        part = RowPartition(csr.shape[0], world)
        for b in batches:
            for seed, step in pairs:
                want, info = S.sample(rows, b, seed, step)
                total = np.zeros_like(want)
                for rank in range(world):
                    lo, hi = part.bounds(rank)
                    got, s_lo, s_hi = owned_call(csr, lo, hi, b, seed, step)
                    assert np.array_equal(got, S.owned(want, info["slots"], s_lo, s_hi)), (world, rank, b, seed, step)
                    total += got
                assert np.array_equal(total, want), (world, b, seed, step)


def check_sharded_world1(csr, batches, pairs):
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.sampler import ShardedTripleSampler
    from tests.test_dist_emu_rowshard_sampler import block_rows
    rows = S.Rows(csr)
    pu = RowPartition(csr.shape[0], 1)
    for seed, step in pairs:
        smp = ShardedTripleSampler(block_rows(csr, pu, 0), pu, 0, device="cuda", seed=seed)
        for b in batches:
            out = torch.full((3, b), -1, dtype=torch.int64, device="cuda")
            smp.sample_into(out, step=step)
            want, _ = S.sample(rows, b, seed, step)
            assert np.array_equal(out.cpu().numpy(), want), (b, seed, step)
        assert bool((smp.claim == 0x7FFFFFFF).all())


def check_full_row_refused():
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.sampler import DeviceTripleSampler, ShardedTripleSampler
    from tests.test_dist_emu_rowshard_sampler import block_rows
    csr = csr_of([[1], [], [0, 1, 2, 3, 4], [2, 3]], 5)
    with pytest.raises(ValueError, match="user 2 "):
        DeviceTripleSampler(csr)
    pu = RowPartition(4, 1)
    with pytest.raises(ValueError, match="user 2 "):
        ShardedTripleSampler(block_rows(csr, pu, 0), pu, 0, device="cuda")


# ----------------------------------------------------------------------------------------------------------------- GPU only

def _grid_n_exist(b):
    return sorted({b, b + 1, math.ceil(1.02 * b), math.ceil(1.1 * b), 2 * b})


@pytest.mark.gpu
def test_one_cta_tiny_n_exist_every_batch():
    for n_exist in (1, 2, 3):
        check_one_cta(sparse_csr(n_exist, n_items=5, seed=n_exist), list(range(1, n_exist + 3)), PAIRS)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 31, 32, 33, 257, 1023, 1024])
def test_one_cta_near_n_exist(b):
    fin = 0
    for n_exist in _grid_n_exist(b):
        fin += check_one_cta(sparse_csr(n_exist, seed=n_exist), [b, min(b + 3, S.ONE_CTA_MAX)], PAIRS)[0]
    if b >= 257:
        assert fin > 0                  # the finish ran and matched


@pytest.mark.gpu
def test_one_cta_baby():
    from mmssl_b200.synthetic import make_dataset
    check_one_cta(make_dataset("baby").train, [1, 31, 32, 33, 257, 1023, 1024], PAIRS)


@pytest.mark.gpu
@pytest.mark.parametrize("n_exist", [1100, 1501])
def test_select_path(n_exist):
    check_multi(sparse_csr(n_exist, seed=n_exist), [1, 7, 1025, n_exist - 1, n_exist, n_exist + 1, 16384], PAIRS)


@pytest.mark.gpu
def test_select_path_baby():
    from mmssl_b200.synthetic import make_dataset
    csr = make_dataset("baby").train
    n_exist = int((np.diff(csr.indptr) > 0).sum())
    check_multi(csr, [1, 7, 1025, n_exist - 1, n_exist, n_exist + 1, 16384], PAIRS_SHORT)


@pytest.mark.gpu
def test_select_path_one_million_users():
    n = 1 << 20
    rng = np.random.default_rng(9)
    csr = sp.csr_matrix((np.ones(n, np.float32), rng.integers(0, 1000, n), np.arange(n + 1)), shape=(n, 1000))
    check_multi(csr, [1, 7, 1025, 16384, n - 1, n, n + 1], PAIRS_SHORT)


@pytest.mark.gpu
def test_edge_rows_both_paths():
    fb = 0
    for csr in (edge_csr(), dense40_csr()):
        n_exist = int((np.diff(csr.indptr) > 0).sum())
        fb += check_one_cta(csr, [1, n_exist - 1, n_exist, n_exist + 1, 1024], PAIRS)[1]
        fb += check_multi(csr, [n_exist, 1025, 4000], PAIRS)
    assert fb > 0                       # the complement fallback ran and matched


@pytest.mark.gpu
def test_items_near_two_to_the_31():
    csr = huge_items_csr()
    check_one_cta(csr, [1, 100, 300, 1024], PAIRS)
    check_multi(csr, [1, 299, 300, 1025], PAIRS)
    check_owned_blocks(csr, [77, 1030], [2], PAIRS_SHORT)


@pytest.mark.gpu
def test_owned_blocks_sum_to_the_batch():
    csr = sparse_csr(700, seed=3)
    n_exist = int((np.diff(csr.indptr) > 0).sum())
    check_owned_blocks(csr, [1, 300, n_exist, 1024, 1025, 2000], [2, 3], PAIRS_SHORT)
    check_owned_blocks(edge_csr(), [7, 1100], [2, 3], PAIRS_SHORT)
    check_owned_blocks(dense40_csr(), [6, 1100], [2, 3], PAIRS_SHORT)


@pytest.mark.gpu
def test_sharded_sampler_world1():
    csr = sparse_csr(1200, seed=4)
    check_sharded_world1(csr, [1, 500, 1024, 1025, 1200], PAIRS)


@pytest.mark.gpu
def test_full_row_refused():
    check_full_row_refused()


@pytest.mark.gpu
def test_one_cta_user_frequencies_chi_square():
    """The one-CTA path at B = 1024 on TikTok, as the multi-CTA test in test_gpu_zz_large_batch.py."""
    from scipy import stats
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("tiktok")
    smp = DeviceTripleSampler(ds.train, seed=19)
    B, steps = 1024, 800
    out = torch.empty(3, B, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(ds.n_users, dtype=torch.int64, device="cuda")
    first = torch.zeros(ds.n_users, dtype=torch.int64, device="cuda")
    for s in range(steps):
        smp.sample_into(out, step=s)
        cnt.index_add_(0, out[0], torch.ones(B, dtype=torch.int64, device="cuda"))
        first.index_add_(0, out[0, :B // 2], torch.ones(B // 2, dtype=torch.int64, device="cuda"))
    exist = smp.exist.cpu().numpy()
    c = cnt.cpu().numpy()
    assert c[np.setdiff1d(np.arange(ds.n_users), exist)].sum() == 0
    c = c[exist].astype(np.float64)
    p = B / len(exist)
    x2 = float((((c - steps * p) ** 2) / (steps * p * (1 - p))).sum())
    assert stats.chi2.sf(x2, len(exist) - 1) > 1e-4 and stats.chi2.cdf(x2, len(exist) - 1) > 1e-4, x2
    f = first.cpu().numpy()[exist].astype(np.float64)
    y2 = float((((f - c / 2) ** 2) / (c / 4)).sum())
    assert stats.chi2.sf(y2, len(exist)) > 1e-4 and stats.chi2.cdf(y2, len(exist)) > 1e-4, y2


@pytest.mark.gpu
def test_positive_and_negative_chi_square_on_device():
    """Every user in every batch (B = n_exist) over a few hundred steps of a 12-item matrix: each (user, item) cell of the row
    expected steps / deg times as a positive, each cell of the complement steps / (12 - deg) times as a negative."""
    from scipy import stats
    from mmssl_b200.sampler import DeviceTripleSampler
    rng = np.random.default_rng(6)
    degs = [1, 2, 3, 5, 6, 8, 10, 11, 4, 7]
    row_lists = [rng.choice(12, size=d, replace=False).tolist() for d in degs]
    csr = csr_of(row_lists, 12)
    smp = DeviceTripleSampler(csr, seed=44)
    steps, n = 600, len(degs)
    pos_c, neg_c = np.zeros((n, 12)), np.zeros((n, 12))
    out = torch.empty(3, n, dtype=torch.int64, device="cuda")
    for s in range(steps):
        u, p, q = smp.sample_into(out, step=s).cpu().numpy()
        np.add.at(pos_c, (u, p), 1)
        np.add.at(neg_c, (u, q), 1)
    x2p = x2n = 0.0
    dfp = dfn = 0
    for u, row in enumerate(row_lists):
        mask = np.zeros(12, bool)
        mask[row] = True
        assert pos_c[u, ~mask].sum() == 0 and neg_c[u, mask].sum() == 0
        ep, en = steps / mask.sum(), steps / (~mask).sum()
        x2p += float(((pos_c[u, mask] - ep) ** 2 / ep).sum()); dfp += int(mask.sum()) - 1
        x2n += float(((neg_c[u, ~mask] - en) ** 2 / en).sum()); dfn += int((~mask).sum()) - 1
    for x2, df in ((x2p, dfp), (x2n, dfn)):
        assert stats.chi2.sf(x2, df) > 1e-4 and stats.chi2.cdf(x2, df) > 1e-4, (x2, df)
