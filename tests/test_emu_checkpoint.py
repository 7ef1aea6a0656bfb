"""Checkpoint and resume (mmssl_b200/checkpoint.py) under the cuemu emulator, where the kernels run in a fixed thread order and
a step is bitwise reproducible: a run that is saved, rebuilt from scratch, loaded and continued must equal the uninterrupted
run bit for bit -- HotStep (injected / generator dropout masks, host / device batches), FullStep across a modality-graph
rebuild with top-k pairs pending, and the Trainer's epoch loop with both samplers."""
import os
import re

import numpy as np
import pytest
import torch

from tests.cuemu import harness

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert bool(torch.equal(a.cpu(), b.cpu())), (what, float((a.double() - b.double()).abs().max()))


# ------------------------------------------------------------------------------------------ HotStep
def _hot_problem():
    from mmssl_b200.synthetic import make_bipartite
    U, I, d, B = 67, 45, 64, 16
    R = make_bipartite(U, I, 420, seed=9).tocsr().astype(np.float32)
    R.sort_indices()
    g = torch.Generator().manual_seed(3)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, 24), "image_trans.bias": torch.randn(d, generator=g) * 0.1, "text_trans.weight": xav(d, 16),
         "text_trans.bias": torch.randn(d, generator=g) * 0.1, "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    feats = (torch.randn(I, 24, generator=g), torch.randn(I, 16, generator=g))
    masks = tuple(((torch.rand(I, d, generator=g) >= 0.2) / 0.8).float() for _ in range(2))
    batches = [(torch.randperm(U, generator=g)[:B], torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g))
               for _ in range(5)]
    return U, I, d, B, R, P, feats, masks, batches


def _hot_step(prob, batches_from, masks_from, P=None):
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import csr_norm
    U, I, d, B, R, P0, feats, masks, _ = prob
    ui, iu = BipartiteGraph.from_scipy(csr_norm(R), device="cpu"), BipartiteGraph.from_scipy(csr_norm(R.T.tocsr()), device="cpu")
    sampler = DeviceTripleSampler(R, device="cpu", seed=4) if batches_from == "device" else None
    hs = HotStep({k: v.clone() for k, v in (P or P0).items()}, tuple(FeatureStore(f.clone()) for f in feats), [ui, iu] * 3,
                 HotStepConfig(embed_size=d, n_layers=2, batch_size=B, proj_impl="simt"), batch=B, sampler=sampler)
    hs.engine.two_streams = False
    if masks_from == "inject":
        hs.masks = masks
    return hs


def _hot_run(hs, prob, steps, first):
    outs = []
    for s in range(first, first + steps):
        if hs.sampler is None:
            hs.set_indices(*prob[-1][s])
        outs.append(hs.run().clone())
    return outs


@pytest.mark.parametrize("batches_from", ["host", "device"])
@pytest.mark.parametrize("masks_from", ["inject", "torch"])
def test_hot_step_resume_is_bitwise_the_uninterrupted_run(monkeypatch, tmp_path, batches_from, masks_from):
    from mmssl_b200 import checkpoint
    from mmssl_b200.engine import LIVE
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    prob = _hot_problem()
    torch.manual_seed(7)
    ref = _hot_step(prob, batches_from, masks_from)
    want = _hot_run(ref, prob, 5, 0)

    torch.manual_seed(7)
    a = _hot_step(prob, batches_from, masks_from)
    _hot_run(a, prob, 3, 0)
    path = str(tmp_path / "hot.ckpt")
    checkpoint.save(dict(a.state_dict(), rng=checkpoint.rng_state("cpu")), path)
    del a
    torch.manual_seed(1234)                                  # another generator state and other parameters: the load restores both
    b = _hot_step(prob, batches_from, masks_from, P={k: torch.randn_like(v) for k, v in prob[5].items()})
    ck = checkpoint.load(path)
    b.load_state_dict(ck)
    checkpoint.set_rng_state(ck["rng"], "cpu")
    got = _hot_run(b, prob, 2, 3)
    for s in range(2):
        _same(got[s], want[3 + s], f"loss step {3 + s}")
    for k in LIVE:
        _same(b.P[k], ref.P[k], k)
        _same(b.m[k], ref.m[k], "m/" + k)
        _same(b.v[k], ref.v[k], "v/" + k)
    _same(b.step_dev, ref.step_dev, "step_dev")
    assert int(b.step_dev[0]) == 5


# ------------------------------------------------------------------------------------------ FullStep
def _fs_draws(c, n):
    g = torch.Generator().manual_seed(11)
    B, I, d = c["B"], c["I"], c["d"]
    mk = lambda rows, w, p: ((torch.rand(rows, w, generator=g) >= p) / (1 - p)).float()
    out = []
    for _ in range(n):
        users = torch.randperm(c["U"], generator=g)[:B]
        pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
        out.append(((users, pos, neg), dict(model_masks=[mk(I, d, c["drop_rate"]) for _ in range(4)],
                                            d_masks1=[mk(2 * B, I // 4, 0.31) for _ in range(4)],
                                            d_masks2=[mk(2 * B, I // 8, 0.5) for _ in range(4)],
                                            gumbel_u=torch.rand(B, I, generator=g), alpha=torch.rand(2 * B, generator=g))))
    return out


def test_full_step_resume_across_a_graph_rebuild_is_bitwise(monkeypatch, tmp_path):
    """T = 2: iterations 0, 1 collect top-k pairs, 2 rebuilds the modality graphs, 3 collects, 4 rebuilds.  The save after
    iteration 3 holds rebuilt graphs and pending pairs; the resumed run must rebuild from exactly those."""
    from mmssl_b200 import checkpoint, gan
    from mmssl_b200.engine import LIVE
    from tests import fullstep_check
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    z, c = fullstep_check.load_trace()
    c = dict(c, T=2)
    draws = _fs_draws(c, 6)

    def run(fs, lo, hi):
        return [{k: v.clone() for k, v in fs.step(*draws[s][0], **draws[s][1]).items() if k != "D_grads"} for s in range(lo, hi)]

    ref, _, _ = fullstep_check.build(z, c, "cpu", proj_impl="simt")
    want = run(ref, 0, 6)
    a, _, _ = fullstep_check.build(z, c, "cpu", proj_impl="simt")
    run(a, 0, 4)
    assert a.pairs["image"] and a.graph_pairs["image"] is not None and a.hs.graphs[2].nnz > 0
    path = str(tmp_path / "full.ckpt")
    checkpoint.save(a.state_dict(), path)
    b, _, _ = fullstep_check.build(z, c, "cpu", proj_impl="simt")
    b.load_state_dict(checkpoint.load(path))
    assert b.idx == 4 and b.hs.graphs[2].nnz == a.hs.graphs[2].nnz
    got = run(b, 4, 6)
    for s in range(2):
        for k in want[4 + s]:
            _same(got[s][k], want[4 + s][k], f"{k} step {4 + s}")
    for k in LIVE:
        _same(b.hs.P[k], ref.hs.P[k], k)
        _same(b.hs.m[k], ref.hs.m[k], "m/" + k)
        _same(b.hs.v[k], ref.hs.v[k], "v/" + k)
    for k in gan.PARAMS + gan.BUFFERS:
        _same(b.D.t[k], ref.D.t[k], "D/" + k)
    for k in gan.PARAMS:
        _same(b.D.m[k], ref.D.m[k], "D.m/" + k)
        _same(b.D.v[k], ref.D.v[k], "D.v/" + k)
    assert b.D.step == ref.D.step == int(b.D.step_dev[0]) == 6


# ------------------------------------------------------------------------------------------ Trainer
_TIME = re.compile(r"\[\d+\.\ds( \+ \d+\.\ds)?\]")


def _trainer(sampler, epochs, seed, lines, ckpt=""):
    from mmssl_b200.dataset import ReferenceDataset
    from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed
    ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
    # the emulated .to("cuda") does not copy: the feature nn.Embedding copies would stay on the loader's read-only arrays
    ds.image_feats, ds.text_feats = np.array(ds.image_feats), np.array(ds.text_feats)
    args = TrainerArgs(dataset="dataset_small", epoch=epochs, batch_size=16, verbose=2, early_stopping_patience=5, m_topk_rate=0.05,
                       Ks="[2, 5, 10]", seed=5, checkpoint=ckpt)
    set_seed(seed)
    return Trainer(ds, args, device="cpu", sampler=sampler, log=lambda s: lines.append(_TIME.sub("[T]", s)))


@pytest.mark.parametrize("sampler", ["reference", "device"])
def test_trainer_resume_equals_the_uninterrupted_run(monkeypatch, tmp_path, sampler):
    import mmssl_b200.Models as M
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    lines_ref = []
    ref = _trainer(sampler, 3, 5, lines_ref)
    ref.train()
    path = str(tmp_path / "run.ckpt")
    lines_a = []
    a = _trainer(sampler, 1, 5, lines_a, ckpt=path)
    a.train()
    assert os.path.exists(path) and not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]
    lines_b = []
    b = _trainer(sampler, 3, 99, lines_b)           # another seed: everything the run depends on comes from the checkpoint
    b.load(path)
    b.train()
    assert lines_a[:-1] + lines_b == lines_ref
    assert b.history == ref.history and len(b.history) == 3
    for (k, x), (k2, y) in zip(sorted(b.model.state_dict().items()), sorted(ref.model.state_dict().items())):
        _same(x, y, k)
    for (k, x), (_, y) in zip(sorted(b.D.state_dict().items()), sorted(ref.D.state_dict().items())):
        _same(x, y, "D/" + k)
    # the model part is the reference's state_dict: fresh modules take it with strict=True
    from mmssl_b200 import checkpoint
    ck = checkpoint.load(path)
    fresh = M.MMSSL(a.n_users, a.n_items, a.args.embed_size, a.weight_size, eval(a.args.mess_dropout), np.asarray(a.data.image_feats),
                    np.asarray(a.data.text_feats))
    fresh.load_state_dict(ck["model"], strict=True)
    d = M.Discriminator(a.n_items)
    d.load_state_dict(ck["D"], strict=True)
    for k, v in ck["model"].items():
        _same(fresh.state_dict()[k], v, k)
