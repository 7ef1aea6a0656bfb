"""The device sampler bit for bit against its exact model, executed on the CPU by the cuemu emulator in both thread orders:
the bodies of tests/test_gpu_zz_sampler_exact.py at small sizes -- the claim finish at B close to n_exist, the select path,
the complement fallback, n_items = 2^31 - 1, the owned entry points block by block, ShardedTripleSampler at world 1, the
full-row refusal."""
import numpy as np
import pytest

from tests import sampler_model as S
from tests import test_gpu_zz_sampler_exact as X
from tests.cuemu import harness


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


def test_one_cta_tiny_and_near_n_exist(emu):
    for n_exist in (1, 2, 3):
        X.check_one_cta(X.sparse_csr(n_exist, n_items=5, seed=n_exist), list(range(1, n_exist + 3)), X.PAIRS)
    fin = 0
    for b, n_exist in ((33, 33), (33, 34), (257, 257), (257, 283), (1024, 1024), (1024, 1045)):
        fin += X.check_one_cta(X.sparse_csr(n_exist, seed=n_exist), [b], X.PAIRS_SHORT)[0]
    assert fin > 0


def test_select_path(emu):
    n_exist = 300
    X.check_multi(X.sparse_csr(n_exist, seed=2), [1, 7, n_exist - 1, n_exist, n_exist + 1, 1025], X.PAIRS)


def test_edge_rows_and_huge_item_ids(emu):
    fb = 0
    for csr in (X.edge_csr(), X.dense40_csr()):
        n_exist = int((np.diff(csr.indptr) > 0).sum())
        fb += X.check_one_cta(csr, [n_exist, n_exist + 1, 40], X.PAIRS_SHORT)[1]
        fb += X.check_multi(csr, [n_exist, 1025], X.PAIRS_SHORT[:1])
    assert fb > 0
    csr = X.huge_items_csr(60)
    X.check_one_cta(csr, [60, 61], X.PAIRS_SHORT)
    X.check_multi(csr, [59, 60], X.PAIRS_SHORT)


def test_owned_blocks_and_world1(emu):
    csr = X.sparse_csr(250, seed=3)
    n_exist = int((np.diff(csr.indptr) > 0).sum())
    X.check_owned_blocks(csr, [n_exist, 1025], [2, 3], X.PAIRS_SHORT[:1])
    X.check_owned_blocks(X.dense40_csr(), [6], [3], X.PAIRS_SHORT[:1])
    X.check_sharded_world1(csr, [n_exist, n_exist + 1, 1025], X.PAIRS_SHORT[:1])


def test_full_row_refused(emu):
    X.check_full_row_refused()
