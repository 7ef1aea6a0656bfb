"""The row-sharded hot step at embedding width 96 on two gloo ranks under the cuemu emulator, both schedules: the body of
tests/test_dist_emu.py with a d = 96 problem (8-lane groups of three float4 in the SpMM and in mmssl_reduce_rows_epilogue)."""
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from tests import test_dist_emu as D

WIDTH = 96


def _problem_w(modal):
    import scipy.sparse as sp
    from mmssl_b200.synthetic import csr_norm, make_bipartite
    U, I, d, B = 203, 131, WIDTH, 48
    r = make_bipartite(U, I, 1500, seed=5)
    g = torch.Generator().manual_seed(2)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, 40), "image_trans.bias": torch.randn(d, generator=g) * 0.1, "text_trans.weight": xav(d, 24),
         "text_trans.bias": torch.randn(d, generator=g) * 0.1, "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    feats = (torch.randn(I, 40, generator=g), torch.randn(I, 24, generator=g))
    masks = tuple(((torch.rand(I, d, generator=g) >= 0.2) / 0.8).float() for _ in range(2))
    users = torch.randperm(U, generator=g)[:B]
    pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
    mods = None
    if modal == "random":
        rng = np.random.default_rng(3)
        mk = lambda nnz: sp.csr_matrix((np.ones(nnz, np.float32), (rng.integers(0, U, nnz), rng.integers(0, I, nnz))), shape=(U, I))
        mods = [(csr_norm(m), csr_norm(m.T.tocsr())) for m in (mk(700), mk(400))]
    return U, I, d, B, csr_norm(r), csr_norm(r.T.tocsr()), P, feats, masks, (users, pos, neg), mods


def _worker(rank, port, modal, schedule, ret):
    D._problem = _problem_w
    D._worker(rank, port, modal, schedule, ret)


@pytest.mark.parametrize("modal,schedule", [("random", "reduce_scatter"), ("random", "allgather")])
def test_row_sharded_hot_step_d96_matches_single_process(modal, schedule):
    port = D._free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(port, modal, schedule, ret), nprocs=D.WORLD, join=True)
    assert len(ret) == D.WORLD
    for rank in range(D.WORLD):
        e = dict(ret[rank])
        gathers, rs = e.pop("gathers_per_step"), e.pop("reduce_scatters_per_step")
        bad = {k: v for k, v in e.items() if not v < 2e-5}
        assert not bad, (rank, bad)
        assert gathers > 0 and (rs > 0) == (schedule == "reduce_scatter")
