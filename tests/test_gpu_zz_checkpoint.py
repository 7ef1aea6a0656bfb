"""Checkpoint and resume on the H100.  A loaded state is bitwise the saved one (tensors, step counter, RNG states), and the
batches and dropout masks drawn after the resume are bitwise those of the uninterrupted run.  The step itself is not bitwise
on the device (heavy-row atomics, DESIGN section 6), so resumed and uninterrupted steps agree to the documented run-to-run
spread: loss terms within 1e-5, gradients within 5e-3 max-norm relative.  A HotStep captured before an in-place load replays
from the loaded state; a Trainer with cuda_graph=True resumes and captures again."""
import os

import numpy as np
import pytest
import torch

from tests.golden_util import rel_err

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
LOSS_TOL, GRAD_TOL = 1e-5, 5e-3


def _problem():
    from mmssl_b200.synthetic import make_bipartite
    U, I, d, B = 3001, 1207, 64, 1024
    R = make_bipartite(U, I, 40000, seed=9).tocsr().astype(np.float32)
    R.sum_duplicates()
    R.data[:] = 1.0
    R.sort_indices()
    g = torch.Generator().manual_seed(3)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, 128), "image_trans.bias": torch.zeros(d), "text_trans.weight": xav(d, 96),
         "text_trans.bias": torch.zeros(d), "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    feats = (torch.randn(I, 128, generator=g), torch.randn(I, 96, generator=g))
    masks = tuple(((torch.rand(I, d, generator=g) >= 0.2) / 0.8).float() for _ in range(2))
    batches = [(torch.randint(0, U, (B,), generator=g), torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g))
               for _ in range(4)]
    return U, I, d, B, R, P, feats, masks, batches


def _step(prob, sampler: bool, P=None):
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import csr_norm
    U, I, d, B, R, P0, feats, _, _ = prob
    ui, iu = BipartiteGraph.from_scipy(csr_norm(R)), BipartiteGraph.from_scipy(csr_norm(R.T.tocsr()))
    smp = DeviceTripleSampler(R, device="cuda", seed=4) if sampler else None
    return HotStep({k: v.cuda().contiguous() for k, v in (P or P0).items()}, tuple(FeatureStore(f.cuda()) for f in feats), [ui, iu] * 3,
                   HotStepConfig(embed_size=d, batch_size=B), batch=B, sampler=smp)


def _recording(hs):
    """Runs steps eagerly and keeps each step's batch, dropout masks, loss terms and gradients."""
    seen = []
    orig = hs._masks

    def masks():
        m = orig()
        seen.append(tuple(t.clone() for t in m))
        return m
    hs._masks = masks

    def run():
        out = hs.run().clone()
        torch.cuda.synchronize()
        return dict(idx=hs.idx.clone(), masks=seen[-1], loss=out, grads={k: g.clone() for k, g in hs.grads.items()})
    return run


def test_resume_restores_the_state_bitwise_and_continues_the_run(tmp_path):
    from mmssl_b200 import checkpoint
    from mmssl_b200.engine import LIVE
    prob = _problem()
    torch.manual_seed(7)
    ref = _recording(_step(prob, sampler=True))
    want = [ref() for _ in range(5)]

    torch.manual_seed(7)
    a = _step(prob, sampler=True)
    run_a = _recording(a)
    for _ in range(3):
        run_a()
    path = str(tmp_path / "hot.ckpt")
    checkpoint.save(dict(a.state_dict(), rng=checkpoint.rng_state("cuda")), path)

    torch.manual_seed(99)
    b = _step(prob, sampler=True, P={k: torch.randn_like(v) for k, v in prob[5].items()})
    ck = checkpoint.load(path)
    b.load_state_dict(ck)
    checkpoint.set_rng_state(ck["rng"], "cuda")
    for k in LIVE:
        assert torch.equal(b.P[k].cpu(), ck["model"][k]), k
        assert torch.equal(b.m[k].cpu(), ck["optim"]["m"][k]), k
        assert torch.equal(b.v[k].cpu(), ck["optim"]["v"][k]), k
    assert int(b.step_dev.cpu()[0]) == ck["optim"]["step"] == 3
    assert torch.equal(torch.get_rng_state(), ck["rng"]["torch"]) and torch.equal(torch.cuda.get_rng_state(), ck["rng"]["cuda"])
    run_b = _recording(b)
    for s in (3, 4):
        got = run_b()
        assert torch.equal(got["idx"], want[s]["idx"]), s                        # the device sampler's batch
        assert all(torch.equal(x, y) for x, y in zip(got["masks"], want[s]["masks"])), s
        e = float(((got["loss"] - want[s]["loss"]).abs() / want[s]["loss"].abs().clamp_min(1e-12)).max())
        assert e < LOSS_TOL, (s, e)
        for k in LIVE:
            assert rel_err(got["grads"][k], want[s]["grads"][k]) < GRAD_TOL, (s, k)


def test_captured_step_replays_from_an_in_place_load(tmp_path):
    from mmssl_b200 import checkpoint
    from mmssl_b200.engine import LIVE
    prob = _problem()
    masks = tuple(m.cuda() for m in prob[7])
    src = _step(prob, sampler=False)
    src.masks = masks
    for s in range(3):
        src.set_indices(*prob[8][s])
        src.run()
    path = str(tmp_path / "src.ckpt")
    checkpoint.save(src.state_dict(), path)
    ck = checkpoint.load(path)

    hs = _step(prob, sampler=False, P={k: torch.randn_like(v) * 0.1 for k, v in prob[5].items()})
    hs.masks = masks
    hs.set_indices(*prob[8][0])
    hs.capture()                                   # recorded on other parameters and moments
    hs.load_state_dict(ck)
    hs.set_indices(*prob[8][3])
    out = hs.replay().clone()
    torch.cuda.synchronize()
    g_replay = {k: g.clone() for k, g in hs.grads.items()}

    eager = _step(prob, sampler=False)
    eager.masks = masks
    eager.load_state_dict(ck)
    eager.set_indices(*prob[8][3])
    want = eager.run().clone()
    e = float(((out - want).abs() / want.abs().clamp_min(1e-12)).max())
    assert e < LOSS_TOL, e
    for k in LIVE:
        assert rel_err(g_replay[k], eager.grads[k]) < GRAD_TOL, k
    assert int(hs.step_dev.cpu()[0]) == int(eager.step_dev.cpu()[0]) == 4


def _fs_draws(c, n, dev="cuda"):
    g = torch.Generator().manual_seed(11)
    B, I, d = c["B"], c["I"], c["d"]
    mk = lambda rows, w, p: (((torch.rand(rows, w, generator=g) >= p) / (1 - p)).float()).to(dev)
    out = []
    for _ in range(n):
        users = torch.randperm(c["U"], generator=g)[:B]
        pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
        out.append(((users.to(dev), pos.to(dev), neg.to(dev)),
                    dict(model_masks=[mk(I, d, c["drop_rate"]) for _ in range(4)], d_masks1=[mk(2 * B, I // 4, 0.31) for _ in range(4)],
                         d_masks2=[mk(2 * B, I // 8, 0.5) for _ in range(4)], gumbel_u=torch.rand(B, I, generator=g).to(dev),
                         alpha=torch.rand(2 * B, generator=g).to(dev))))
    return out


def _fs_tensors(fs):
    """Every tensor of a FullStep's training state, by name."""
    from mmssl_b200 import gan
    from mmssl_b200.engine import LIVE
    t = {}
    for k in LIVE:
        t["P/" + k], t["m/" + k], t["v/" + k] = fs.hs.P[k], fs.hs.m[k], fs.hs.v[k]
    for k in gan.PARAMS + gan.BUFFERS:
        t["D/" + k] = fs.D.t[k]
    for k in gan.PARAMS:
        t["Dm/" + k], t["Dv/" + k] = fs.D.m[k], fs.D.v[k]
    t["step_dev"], t["D.step_dev"] = fs.hs.step_dev, fs.D.step_dev
    return t


def test_full_step_load_is_bitwise_and_keeps_or_drops_the_captured_iteration(tmp_path):
    from mmssl_b200 import checkpoint
    from tests import fullstep_check
    z, c = fullstep_check.load_trace()
    draws = _fs_draws(c, 6)
    early = str(tmp_path / "early.ckpt")
    steady = str(tmp_path / "steady.ckpt")
    a, _, _ = fullstep_check.build(z, c, "cuda")
    a.step(*draws[0][0], **draws[0][1])
    assert a.pairs["image"]                          # top-k pairs pending, the modality graphs still the training graphs
    checkpoint.save(a.state_dict(), early)
    for s in (1, 2):
        a.step(*draws[s][0], **draws[s][1])
    assert a.steady()
    a.capture()
    a.step(*draws[3][0], **draws[3][1])              # a replay
    checkpoint.save(a.state_dict(), steady)
    ck = checkpoint.load(steady)

    # the loaded state is bitwise the saved one: every tensor, both step counters of D, the bookkeeping
    b, _, _ = fullstep_check.build(z, c, "cuda")
    b.load_state_dict(ck)
    torch.cuda.synchronize()
    want = {**{"P/" + k: v for k, v in ck["model"].items()}, **{"m/" + k: v for k, v in ck["optim"]["m"].items()},
            **{"v/" + k: v for k, v in ck["optim"]["v"].items()}, **{"D/" + k: v for k, v in ck["D"].items()},
            **{"Dm/" + k: v for k, v in ck["D_optim"]["m"].items()}, **{"Dv/" + k: v for k, v in ck["D_optim"]["v"].items()},
            "step_dev": torch.tensor([ck["optim"]["step"]], dtype=torch.int32),
            "D.step_dev": torch.tensor([ck["D_optim"]["step"]], dtype=torch.int32)}
    for k, t in _fs_tensors(b).items():
        assert torch.equal(t.cpu(), want[k].view_as(t.cpu())), k
    assert b.D.step == int(b.D.step_dev.cpu()[0]) == ck["D_optim"]["step"] == a.D.step == 5      # 4 iterations + the capture's warm-up
    assert b.idx == a.idx == 5 and b.pairs == {"image": [], "text": []} and b.hs.graphs[2].nnz == 0

    # same modality graphs: the captured iteration is kept; other graphs: it is dropped and the training graphs are back
    a.load_state_dict(ck)
    assert a._graph is not None
    a.load_state_dict(checkpoint.load(early))
    assert a._graph is None and a.hs.graphs[2] is a.hs.graphs[0] and a.idx == 1 and len(a.pairs["image"]) == 1


def test_capture_keeping_the_state_trains_nothing(tmp_path):
    from mmssl_b200 import checkpoint
    from tests import fullstep_check
    z, c = fullstep_check.load_trace()
    draws = _fs_draws(c, 3)
    fs, _, _ = fullstep_check.build(z, c, "cuda")
    for s in range(3):
        fs.step(*draws[s][0], **draws[s][1])
    before = {k: v.clone() for k, v in _fs_tensors(fs).items()}
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state())
    d_step, idx = fs.D.step, fs.idx
    fs.capture(keep_state=True)
    torch.cuda.synchronize()
    assert fs._graph is not None and fs.D.step == d_step and fs.idx == idx
    for k, t in _fs_tensors(fs).items():
        assert torch.equal(t, before[k]), k
    assert torch.equal(torch.get_rng_state(), rng[0]) and torch.equal(torch.cuda.get_rng_state(), rng[1])


def test_trainer_with_cuda_graph_resumes_and_captures_again(tmp_path):
    """The uninterrupted run captured in epoch 0 (its capture's warm-up iteration is in the saved state); the resumed run captures
    again without training an extra iteration: the optimiser step counters, BatchNorm batch counts and sampler position end
    where the uninterrupted run's do."""
    from mmssl_b200.dataset import ReferenceDataset
    from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed
    ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
    path = str(tmp_path / "run.ckpt")
    mk = lambda epochs, ck="", seed=5: TrainerArgs(dataset="dataset_small", epoch=epochs, batch_size=16, verbose=1,
                                                  early_stopping_patience=5, m_topk_rate=0.05, Ks="[2, 5, 10]", seed=seed, checkpoint=ck)
    set_seed(5)
    ref = Trainer(ds, mk(3), sampler="device", log=None, cuda_graph=True)
    ref.train()
    set_seed(5)
    a = Trainer(ds, mk(1, path), sampler="device", log=None, cuda_graph=True)
    a.train()
    assert a.step._graph is not None
    with pytest.raises(ValueError, match="sampler_seed"):
        Trainer(ds, mk(3, seed=6), sampler="device", log=None, cuda_graph=True).load(path)
    set_seed(99)
    b = Trainer(ds, mk(3), sampler="device", log=None, cuda_graph=True)
    b.load(path)
    assert b.step._graph is None and b.history == a.history and b._n_sampled == a._n_sampled
    b.train()
    assert b.step._graph is not None                                  # captured again once the modality graphs settled
    assert [h["epoch"] for h in b.history] == [0, 1, 2] and b.history[0] == a.history[0]
    assert all(np.isfinite(h["loss"]) for h in b.history)
    assert b._n_sampled == ref._n_sampled == 3 * a._n_sampled
    assert b.step.D.step == ref.step.D.step == int(b.step.D.step_dev.cpu()[0])
    assert int(b.step.hs.step_dev.cpu()[0]) == int(ref.step.hs.step_dev.cpu()[0])
    assert int(b.D.net[2].num_batches_tracked) == int(ref.D.net[2].num_batches_tracked)
