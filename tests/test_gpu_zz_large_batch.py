"""Device sampler at any batch size (csrc/sampler.cu, multi-CTA radix select above 1024 triples) and the training step with
it: the semantics of Data.sample (load_data.py:153-191), determinism in (seed, step, batch), fresh batches across CUDA-graph
replays, and one captured hot step at B = 4096 against the CPU oracle.  The check_* bodies also run in the emulator
(tests/test_emu_large_batch.py)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.golden_util import rel_err


def random_csr(n_users, n_items, seed, empty_every=7):
    """Rows of 1..8 sorted items; every `empty_every`-th user has none (not eligible)."""
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for u in range(n_users):
        if u % empty_every == 3:
            continue
        items = rng.choice(n_items, size=int(rng.integers(1, 9)), replace=False)
        rows += [u] * len(items)
        cols += items.tolist()
    return sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_users, n_items))


def sample_multi(smp, batch, step=0, step_dev=None):
    """The multi-CTA entry point called directly, at any batch size (the sampler class routes batches of up to 1024
    triples to the one-CTA kernel)."""
    from mmssl_b200 import _lib
    from mmssl_b200._lib import ptr, stream
    lib = _lib.load(require_device=True)
    n_exist = smp.exist.numel()
    nbytes = lib.mmssl_sampler_workspace_bytes(n_exist, batch)
    ws = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    out = torch.empty(3, batch, dtype=torch.int64, device="cuda")
    _lib.check(lib.mmssl_sample_triples_multi(ptr(smp.indptr), ptr(smp.indices), ptr(smp.exist), n_exist, smp.n_items, batch, smp.seed,
                                              ptr(step_dev), int(step), ptr(ws), ws.numel(), ptr(out[0]), ptr(out[1]), ptr(out[2]),
                                              stream()))
    torch.cuda.synchronize()
    if nbytes:      # the select's block counter and histogram (SelectState.arrive, .hist) are left zero for the next call
        assert int(ws[24:28].count_nonzero()) == 0 and int(ws[32:32 + 4 * 256].count_nonzero()) == 0
    return out


def check_triples(csr, out, distinct):
    """Users with >= 1 item (distinct when asked), positives in the user's row, negatives outside it."""
    u, p, n = (np.array(t.cpu().numpy(), dtype=np.int64) for t in out)
    deg = np.diff(csr.indptr)
    assert (deg[u] > 0).all()
    if distinct:
        assert len(np.unique(u)) == len(u)
    n_items = csr.shape[1]
    pairs = np.repeat(np.arange(csr.shape[0], dtype=np.int64), deg) * n_items + csr.indices
    assert np.isin(u * n_items + p, pairs).all()
    assert not np.isin(u * n_items + n, pairs).any()
    assert (n >= 0).all() and (n < n_items).all()


def check_multi_semantics(csr, batches, seed=7):
    """Every batch size up to n_exist (including n_exist: a permutation) gives distinct users; larger ones draw with
    replacement.  Equal (seed, step, batch) give bitwise equal batches; other steps differ."""
    from mmssl_b200.sampler import DeviceTripleSampler
    smp = DeviceTripleSampler(csr, seed=seed)
    n_exist = smp.exist.numel()
    for b in batches:
        out = sample_multi(smp, b, step=3)
        check_triples(csr, out, distinct=b <= n_exist)
        if b == n_exist:
            assert np.array_equal(np.sort(out[0].cpu().numpy()), smp.exist.cpu().numpy())
        again = sample_multi(smp, b, step=3)
        assert torch.equal(out, again)
        if b >= 16:
            assert not torch.equal(out[0], sample_multi(smp, b, step=4)[0])
    # the device step counter gives the same batch as the host step
    step = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    b = batches[0]
    assert torch.equal(sample_multi(smp, b, step_dev=step), sample_multi(smp, b, step=5))


def check_class_routing(csr, big):
    """sample_into takes the one-CTA kernel up to 1024 triples and the multi-CTA path above; the latter equals the direct call."""
    from mmssl_b200 import _lib
    from mmssl_b200.sampler import DeviceTripleSampler
    smp = DeviceTripleSampler(csr, seed=3)
    log = []
    _lib.call_log = log
    try:
        out = torch.empty(3, 1024, dtype=torch.int64, device="cuda")
        smp.sample_into(out, step=2)
        assert log == ["mmssl_sample_triples"] or log == []      # (the emulator's library is not counted)
        del log[:]
        big_out = torch.empty(3, big, dtype=torch.int64, device="cuda")
        smp.sample_into(big_out, step=2)
        assert log == ["mmssl_sample_triples_multi"] or log == []
    finally:
        _lib.call_log = None
    check_triples(csr, out, distinct=True)
    check_triples(csr, big_out, distinct=big <= smp.exist.numel())
    assert torch.equal(big_out, sample_multi(smp, big, step=2))


# ----------------------------------------------------------------------------------------------------------------- GPU only

@pytest.mark.gpu
def test_multi_sampler_semantics_tiktok():
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("tiktok")
    n_exist = int((np.diff(ds.train.indptr) > 0).sum())
    check_multi_semantics(ds.train, [1025, 2048, 4096, n_exist - 1, n_exist, n_exist + 1, 16384, 1, 100, 1024])


@pytest.mark.gpu
def test_multi_sampler_semantics_baby_full_permutation():
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("baby")
    n_exist = int((np.diff(ds.train.indptr) > 0).sum())
    check_multi_semantics(ds.train, [16384, n_exist])


@pytest.mark.gpu
def test_sampler_routing():
    from mmssl_b200.synthetic import make_dataset
    check_class_routing(make_dataset("tiktok").train, 4096)


@pytest.mark.gpu
def test_multi_sampler_user_frequencies_chi_square():
    """Over S steps every eligible user is drawn Binomial(S, B / n_exist) times when each step is a uniform B-subset."""
    from scipy import stats
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("tiktok")
    smp = DeviceTripleSampler(ds.train, seed=19)
    B, S = 2048, 400
    out = torch.empty(3, B, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(ds.n_users, dtype=torch.int64, device="cuda")
    first = torch.zeros(ds.n_users, dtype=torch.int64, device="cuda")     # how often a user lands in the first half of a batch
    for s in range(S):
        smp.sample_into(out, step=s)
        cnt.index_add_(0, out[0], torch.ones(B, dtype=torch.int64, device="cuda"))
        first.index_add_(0, out[0, :B // 2], torch.ones(B // 2, dtype=torch.int64, device="cuda"))
    exist = smp.exist.cpu().numpy()
    c = cnt.cpu().numpy()
    assert c[np.setdiff1d(np.arange(ds.n_users), exist)].sum() == 0
    c = c[exist].astype(np.float64)
    p = B / len(exist)
    x2 = float((((c - S * p) ** 2) / (S * p * (1 - p))).sum())
    assert stats.chi2.sf(x2, len(exist) - 1) > 1e-3, x2
    assert stats.chi2.cdf(x2, len(exist) - 1) > 1e-3, x2         # not suspiciously even either
    # the order inside a batch is random too: each time a user is drawn it lands in the first half with probability 1/2
    f = first.cpu().numpy()[exist].astype(np.float64)
    y2 = float((((f - c / 2) ** 2) / (c / 4)).sum())
    assert stats.chi2.sf(y2, len(exist) - 1) > 1e-3, y2


@pytest.mark.gpu
def test_multi_sampler_replays_fresh_batches_in_a_cuda_graph():
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("tiktok")
    smp = DeviceTripleSampler(ds.train, seed=23)
    B = 4096
    smp.reserve(B)
    out = torch.empty(3, B, dtype=torch.int64, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        smp.sample_into(out, step_dev=step)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        smp.sample_into(out, step_dev=step)
    got = []
    for k in range(4):
        step.fill_(k)
        g.replay()
        torch.cuda.synchronize()
        got.append(out.clone())
    ref = torch.empty_like(out)
    for k in range(4):
        smp.sample_into(ref, step=k)
        assert torch.equal(got[k], ref)
        check_triples(ds.train, got[k], distinct=True)
    assert not torch.equal(got[0][0], got[1][0])


@pytest.mark.gpu
def test_captured_hot_step_at_4096_with_device_sampler_vs_oracle():
    """One HotStep at B = 4096 with the device sampler, captured in a CUDA graph: the five loss terms and every live parameter
    gradient against the CPU oracle on the triples the graph drew, 1e-4."""
    import bench
    from oracle import mmssl_oracle as O
    from mmssl_b200.engine import LIVE
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.sampler import DeviceTripleSampler
    torch.set_num_threads(8)
    dev = torch.device("cuda")
    batch = 4096
    ds, P, feats, graphs, feats_cpu = bench.build_problem("baby", 2022, dev)
    cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=batch)
    smp = DeviceTripleSampler(ds.train, device=dev, seed=31)
    hs = HotStep({k: v.clone() for k, v in P.items()}, feats, graphs, cfg, batch=batch, optimizer_step=False, sampler=smp)
    g = torch.Generator().manual_seed(5)
    masks = tuple((torch.rand(ds.n_items, ds.embed_size, generator=g) >= 0.2).float() / 0.8 for _ in range(2))
    hs.masks = tuple(m.cuda() for m in masks)
    hs.capture(warmup=1)
    hs.step_dev.fill_(7)
    out5 = hs.replay().clone().cpu()
    torch.cuda.synchronize()
    users, pos, neg = (t.cpu() for t in hs.idx)
    check_triples(ds.train, hs.idx, distinct=True)
    ref = torch.empty_like(hs.idx)
    smp.sample_into(ref, step=7)
    assert torch.equal(ref, hs.idx)
    ui, iu = O.to_torch_coo(ds.ui_norm), O.to_torch_coo(ds.iu_norm)
    ocfg = O.HotPathConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=batch)
    po = {k: v.cpu().clone().requires_grad_(True) for k, v in P.items()}
    outs = O.forward_closed(po, feats_cpu[0], feats_cpu[1], (ui, iu, ui, iu, ui, iu), ocfg, dropout_masks=masks)
    total, parts = O.hot_loss(outs, users.numpy(), pos.numpy(), neg.numpy(), ds.n_items, ocfg)
    total.backward()
    for got, want in zip(out5.tolist(), [float(total), float(parts["mf"]), float(parts["emb"]), float(parts["feat_reg"]), float(parts["cl"])]):
        assert abs(got - want) <= 1e-4 * max(abs(want), 1e-12), (got, want)
    for k in LIVE:
        assert rel_err(hs.grads[k], po[k].grad) < 1e-4, (k, rel_err(hs.grads[k], po[k].grad))


def reference_dataset(n_users, n_items, seed):
    """A ReferenceDataset built in memory from random_csr: one held-out test and one validation item per eligible user."""
    from mmssl_b200.dataset import ReferenceDataset
    rng = np.random.default_rng(seed)
    csr = random_csr(n_users, n_items, seed)
    train, test, val = {}, {}, {}
    for u in range(n_users):
        row = csr.indices[csr.indptr[u]:csr.indptr[u + 1]].tolist()
        if not row:
            continue
        train[u] = row
        free = np.setdiff1d(np.arange(n_items), row)
        t, v = rng.choice(free, size=2, replace=False)
        test[u], val[u] = [int(t)], [int(v)]
    feats = lambda w: rng.standard_normal((n_items, w)).astype(np.float32)
    return ReferenceDataset(n_users, n_items, csr.nnz, len(test), sorted(train), train, test, val, csr, feats(96), feats(48))


def run_trainer_epochs(ds, batch, epochs=2):
    """Trainer with the device sampler: finite losses and metrics; returns the trainer."""
    from mmssl_b200.trainer import Trainer, TrainerArgs, set_seed
    args = TrainerArgs(dataset="in_memory", epoch=epochs, batch_size=batch, verbose=1, early_stopping_patience=5, m_topk_rate=0.05,
                       Ks="[2, 5, 10]", seed=5)
    set_seed(args.seed)
    tr = Trainer(ds, args, device="cuda", sampler="device", log=lambda *_: None)
    best, _ = tr.train()
    assert len(tr.history) == epochs
    assert all(np.isfinite([h["loss"], h["mf_loss"], h["emb_loss"], h["recall"], h["ndcg"]]).all() for h in tr.history)
    ret = tr.test(list(ds.test_set.keys()), is_val=False)
    assert all(np.isfinite(np.asarray(ret[k], dtype=np.float64)).all() for k in ("recall", "precision", "ndcg", "hit_ratio"))
    assert 0.0 <= best <= 1.0
    return tr


@pytest.mark.gpu
def test_trainer_epoch_with_device_sampler_at_4096():
    """A batch of 4096 on the small golden dataset (61 users): the device sampler draws it with replacement."""
    import os
    from mmssl_b200.dataset import ReferenceDataset
    ds = ReferenceDataset.load(os.path.join(os.path.dirname(__file__), "golden", "dataset_small"))
    run_trainer_epochs(ds, 4096)


@pytest.mark.gpu
def test_trainer_epochs_with_device_sampler_select_path():
    """A batch of 1500 out of 1714 eligible users: every Trainer batch goes through the multi-CTA radix select (distinct
    users) and the epochs finish with finite losses and metrics."""
    from mmssl_b200 import _lib
    ds = reference_dataset(2000, 400, seed=4)
    assert 1024 < 1500 < len(ds.exist_users)
    log = []
    _lib.call_log = log
    try:
        tr = run_trainer_epochs(ds, 1500)
    finally:
        _lib.call_log = None
    assert "mmssl_sample_triples_multi" in log and "mmssl_sample_triples" not in log
    users, pos, neg = tr.sample()
    check_triples(ds.train_mat, torch.stack([users, pos, neg]), distinct=True)
