"""The exact sampler model (tests/sampler_model.py) is a correct specification of the device sampler: it reproduces batches the
kernels drew (tests/golden/device_sampler_batches.npz), and the batches it describes have the distribution of the reference's
Data.sample (load_data.py:153-191) -- distinct users drawn uniformly in a uniform order, positives uniform over the row,
negatives uniform over the complement, on both slot paths and through the claim finish and the complement fallback.
Fixed seeds make every statistic deterministic; both tails of each chi-square are held above 1e-4."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy import stats

from tests import sampler_model as S

GOLD = os.path.join(os.path.dirname(__file__), "golden", "device_sampler_batches.npz")


def rows_of(row_lists, n_items):
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in row_lists])])
    indices = np.concatenate([np.sort(np.asarray(r, np.int64)) for r in row_lists]) if indptr[-1] else np.zeros(0, np.int64)
    return S.Rows.from_arrays(indptr, indices, n_items)


def one_item_rows(n_exist, n_items=50, seed=0):
    rng = np.random.default_rng(seed)
    return rows_of([[int(i)] for i in rng.integers(0, n_items, n_exist)], n_items)


def both_tails(x2, df, what):
    lo, hi = stats.chi2.cdf(x2, df), stats.chi2.sf(x2, df)
    assert lo > 1e-4 and hi > 1e-4, (what, x2, df, lo, hi)


# ------------------------------------------------------------------------------------------------------------ kernel bits
def test_model_reproduces_recorded_kernel_batches():
    g = np.load(GOLD)
    meta = json.loads(bytes(g["meta"]).decode())
    assert {m["path"] for m in meta} == {"one", "multi"} and len({m["seed"] for m in meta}) == 4
    for m in meta:
        name = m["matrix"]
        rows = S.Rows.from_arrays(g[f"{name}_indptr"], g[f"{name}_indices"], g[f"{name}_shape"][1])
        fn = S.one_cta if m["path"] == "one" else S.multi
        out, info = fn(rows, m["batch"], int(m["seed"]), m["step"])
        assert info["finish"] == 0 and info["fallback"] == 0, m        # the recorded batches avoid both new branches
        np.testing.assert_array_equal(out, g[m["key"]], err_msg=str(m))


def test_rng_reference_values():
    """splitmix64 of 0 and 1 (the published constants of the generator), and below() at the ends of its range."""
    assert int(S.splitmix64(0)) == 0xE220A8397B1DCDAF
    assert int(S.splitmix64(1)) == 0x910A2DEC89025CC1
    assert int(S.below(0xFFFFFFFF, 7)) == 6 and int(S.below(0, 7)) == 0
    assert int(S.below(0xFFFFFFFF, 2 ** 31 - 1)) == 2 ** 31 - 2
    assert S.slot_bits(1) == 1 and S.slot_bits(2) == 1 and S.slot_bits(3) == 2 and S.slot_bits(1025) == 11


# ------------------------------------------------------------------------------------------------------------ users
@pytest.mark.parametrize("n_exist", [1, 2, 3, 31, 32, 33, 64, 257])
def test_distinct_users_at_every_batch_up_to_n_exist(n_exist):
    rows = one_item_rows(n_exist)
    for b in range(1, n_exist + 1):
        for step in (0, 1):
            out, _ = S.one_cta(rows, b, 7, step)
            assert len(np.unique(out[0])) == b, (b, step)
            out, _ = S.multi(rows, b, 7, step)
            assert len(np.unique(out[0])) == b, (b, step)


def test_distinct_users_near_n_exist_through_the_finish():
    """B close to n_exist at B = 1024: the claim rounds leave threads pending, the finish serves them with distinct slots."""
    finish = 0
    for n_exist in (1024, 1025, 1029, 1045, 1127):
        rows = one_item_rows(n_exist)
        for step in range(3):
            slots, draws, info = S.claim_slots(2022, step, n_exist, 1024)
            assert len(np.unique(slots)) == 1024 and slots.min() >= 0 and slots.max() < n_exist
            finish += info["finish"]
    assert finish > 0


@pytest.mark.parametrize("path", ["one", "multi"])
@pytest.mark.parametrize("ratio", [1.0, 0.99, 0.9, 0.5, 0.05])
def test_users_and_positions_uniform(path, ratio):
    """Over S batches each slot is drawn Binomial(S, B / n_exist) times, and each time lands in the first half of the batch
    with probability 1/2 (B = n_exist: every batch is a permutation, only the order is random)."""
    B = 256
    n_exist = int(round(B / ratio))
    steps = 400
    cnt, first = np.zeros(n_exist), np.zeros(n_exist)
    fin = 0
    for step in range(steps):
        if path == "one":
            slots, _, info = S.claim_slots(91, step, n_exist, B)
            fin += info["finish"]
        else:
            slots, _ = S.select_slots(91, step, n_exist, B)
        assert len(np.unique(slots)) == B
        np.add.at(cnt, slots, 1)
        np.add.at(first, slots[:B // 2], 1)
    if path == "one" and ratio >= 0.99:
        assert fin > 0                              # the statistic covers the finish
    p = B / n_exist
    if p < 1:
        both_tails(float(((cnt - steps * p) ** 2 / (steps * p * (1 - p))).sum()), n_exist - 1, "users")
    both_tails(float(((first - cnt / 2) ** 2 / (cnt / 4)).sum()), n_exist, "positions")


# ------------------------------------------------------------------------------------------------------------ positives, negatives
def test_positives_uniform_over_each_row():
    """Every slot in every batch (B = n_exist): cell (user, item) expected steps / deg >= 50 times."""
    rng = np.random.default_rng(4)
    row_lists = [rng.choice(30, size=d, replace=False).tolist() for d in (1, 2, 3, 5, 6, 4, 2, 6)]
    rows = rows_of(row_lists, 30)
    steps = 300
    hits = {}
    for step in range(steps):
        out, _ = S.one_cta(rows, rows.n_exist, 5, step)
        for u, p in zip(out[0], out[1]):
            hits[(int(u), int(p))] = hits.get((int(u), int(p)), 0) + 1
    x2, df = 0.0, 0
    for u, row in enumerate(row_lists):
        assert sum(hits.get((u, i), 0) for i in row) == steps
        assert all(k[1] in row for k in hits if k[0] == u)
        if len(row) > 1:
            e = steps / len(row)
            x2 += sum((hits.get((u, i), 0) - e) ** 2 / e for i in row)
            df += len(row) - 1
    both_tails(x2, df, "positives")


def _negatives(row, n_items, n, seed=3):
    """n independent negatives of one user (threads 0..n-1 all drawing for slot 0), and the fallback count."""
    rows = rows_of([row], n_items)
    out, fb = S.draw_triples(rows, np.zeros(n, np.int64), np.zeros(n, np.int64), seed, 1)
    return out[2], fb


@pytest.mark.parametrize("n_items,missing", [
    (40, [17]), (40, [0, 20, 39]), (12, [0, 1, 5, 6, 11]),
    (50_000, [0]), (50_000, [49_999]), (50_000, [25_000]), (50_000, [0, 25_000, 49_999]), (50_000, [1, 2, 49_998])])
def test_negatives_uniform_over_the_complement(n_items, missing):
    """Rows missing a few items: negatives only ever outside the row and uniform over the missing items.  At 50 000 items the
    4096 rejection draws mostly fail and the complement fallback takes over."""
    row = np.setdiff1d(np.arange(n_items), missing)
    n = 150 * len(missing)
    neg, fb = _negatives(row, n_items, n)
    assert np.isin(neg, missing).all()
    if n_items == 50_000:
        assert fb > n // 2
    if len(missing) > 1:
        c = np.array([(neg == m).sum() for m in missing], np.float64)
        e = n / len(missing)
        both_tails(float(((c - e) ** 2 / e).sum()), len(missing) - 1, "negatives")


def test_negatives_uniform_for_sparse_rows():
    row = [3, 4, 9]
    neg, fb = _negatives(row, 20, 17 * 200)
    assert fb == 0 and not np.isin(neg, row).any()
    c = np.bincount(neg, minlength=20)[np.setdiff1d(np.arange(20), row)].astype(np.float64)
    both_tails(float(((c - 200) ** 2 / 200).sum()), 16, "negatives")


def test_complement_fallback_is_the_jth_missing_item():
    """The fallback's rank search against a direct enumeration of the complement, for every j of a few rows."""
    for row, n_items in (([0, 1, 2], 5), ([1, 3], 6), ([0, 2, 3, 7, 8, 9], 10), ([], 4), ([5], 6)):
        row = np.asarray(row, np.int64)
        missing = np.setdiff1d(np.arange(n_items), row)
        for j in range(len(missing)):
            m = int(np.searchsorted(row - np.arange(len(row)), j, side="right"))
            assert j + m == missing[j], (row, j)


def test_owned_blocks_sum_to_the_batch():
    rows = one_item_rows(300)
    for b in (50, 300, 1100):
        out, info = S.sample(rows, b, 8, 2)
        bounds = [0, 97, 180, 300]
        parts = [S.owned(out, info["slots"], lo, hi) for lo, hi in zip(bounds[:-1], bounds[1:])]
        np.testing.assert_array_equal(sum(parts), out)
