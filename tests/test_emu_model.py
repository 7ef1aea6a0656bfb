"""The whole hot path on the CPU: drop-in ``Models.MMSSL`` (autograd wrappers), the fused ``HotStep`` and three AdamW steps,
executed by the cuemu fiber emulator (tests/cuemu) against the golden vectors minted from the unmodified reference -- the
bodies of tests/test_gpu_model.py.  The wgmma GEMM is replaced by a host statement of its contract
(tests/cuemu/gemm_bf16x3_host.cpp: bf16 hi/lo operands, split-K partials), every other kernel is the real source."""
import pytest

from tests import test_gpu_model as M
from tests.cuemu import harness
from tests.golden_util import CASES, Golden, rel_err


@pytest.fixture
def emu(monkeypatch):
    harness.set_order("fwd")
    return harness.emulated_device(monkeypatch)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("proj_impl", ["tc", "simt"])
def test_model_forward_backward(emu, case, proj_impl):
    M.test_model_forward_backward_vs_reference(case, proj_impl)


@pytest.mark.parametrize("case", CASES)
def test_fused_hot_step(emu, case):
    M.test_fused_hot_step_vs_reference(case)


def test_three_adamw_steps_vs_oracle(emu):
    """tests/test_gpu_model.py::test_hot_step_graph_replay_and_adamw_vs_oracle without the CUDA graph."""
    from oracle import mmssl_oracle as O
    g = Golden("case_train_rand_k3")
    hs, P = M._hotstep(g, optimizer_step=True)
    cpu = O.CpuHotStep({k: v.clone() for k, v in g.params.items()}, g.image_feats, g.text_feats, g.graphs(), g.cfg["I"], g.oracle_cfg())
    got = [float(hs.run()[0]) for _ in range(3)]
    want = [cpu.step(g.users, g.pos, g.neg, dropout_masks=g.masks) for _ in range(3)]
    for a, b in zip(got, want):
        assert abs(a - b) < M.TOL * abs(b)
    for k in M.LIVE:
        assert rel_err(P[k], cpu.params[k]) < M.TOL, k
    assert int(hs.step_dev) == 3


@pytest.mark.parametrize("d,modal", [(128, "random"), (256, "random"), (128, "alias")])
def test_other_widths(emu, d, modal):
    M.test_hot_step_other_widths_vs_oracle(d, modal)


def test_hot_step_batch_beyond_one_infonce_block(emu):
    """B = 1300 triples: more than one 1024-row block of the reference's batched_contrastive_loss (main.py:228-246) and not a
    multiple of it (SURVEY 8d's second column uses B = 16384): loss terms and all live gradients of the fused step vs the oracle."""
    import torch
    from oracle import mmssl_oracle as O
    from mmssl_b200.engine import LIVE, FeatureStore
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.synthetic import csr_norm, make_bipartite
    U, I, d, B = 1500, 300, 64, 1300
    r = make_bipartite(U, I, 7000, seed=1)
    g = torch.Generator().manual_seed(0)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, 24), "image_trans.bias": torch.zeros(d), "text_trans.weight": xav(d, 16), "text_trans.bias": torch.zeros(d),
         "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d),
         "weight_dict.w_q": xav(d, d), "weight_dict.w_k": xav(d, d)}
    feats = (torch.randn(I, 24, generator=g), torch.randn(I, 16, generator=g))
    users, pos, neg = torch.randperm(U, generator=g)[:B], torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
    cfg = HotStepConfig(embed_size=d, n_layers=2, batch_size=B, drop_rate=0.0, proj_impl="simt")
    gu, gi = BipartiteGraph.from_scipy(csr_norm(r), device="cpu"), BipartiteGraph.from_scipy(csr_norm(r.T.tocsr()), device="cpu")
    hs = HotStep({k: v.clone() for k, v in P.items()}, tuple(FeatureStore(f) for f in feats), [gu, gi, gu, gi, gu, gi], cfg, batch=B,
                 optimizer_step=False)
    hs.set_indices(users, pos, neg)
    out = hs.run().clone()
    ocfg = O.HotPathConfig(embed_size=d, n_layers=2, batch_size=B, drop_rate=0.0)
    params = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    ui, iu = O.build_graphs(r)
    outs = O.forward_closed(params, feats[0], feats[1], (ui, iu, ui, iu, ui, iu), ocfg, dropout_masks=None, training=False)
    total, parts = O.hot_loss(outs, users, pos, neg, I, ocfg)
    total.backward()
    want = [float(total.detach()), float(parts["mf"].detach()), float(parts["emb"].detach()), float(parts["feat_reg"].detach()), float(parts["cl"].detach())]
    for a, b in zip(out.tolist(), want):
        assert abs(a - b) <= 1e-4 * max(abs(b), 1e-12)
    for k in LIVE:
        assert rel_err(hs.grads[k], params[k].grad) < 1e-4, k
