"""sampler.ShardedTripleSampler at world sizes 2 and 3 over gloo, every rank running the REAL sampler kernels under the cuemu
emulator: every rank's [3, B] batch is bitwise DeviceTripleSampler's on the whole training matrix -- both paths (one CTA up to
1024 triples, the radix select above), a permutation (B = n_exist), with replacement (B > n_exist), several steps, odd user
counts (the last block padded), users without training items in every block, a rank whose block has no such user at all and
batches whose users all lie in one block.  Also: the chain write_shards -> ShardedDataset -> ShardedTripleSampler,
RowShardedHotStep(sampler=...) against the same step fed by set_indices, and a world-2 checkpoint of a sampled run resumed
at world 1 by HotStep with DeviceTripleSampler."""
import os
import socket

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SEED = 77


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class _MP:
    def setattr(self, o, n, v):
        setattr(o, n, v)


def _init(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from tests.cuemu import harness
    harness.set_order("fwd")
    harness.emulated_device(_MP())


def _matrix(U, I, nonempty, density, seed):
    """[U, I] training pattern whose non-empty rows are exactly `nonempty` (bool [U]), sorted rows."""
    rng = np.random.default_rng(seed)
    dense = rng.random((U, I)) < density
    dense[np.arange(U), rng.integers(0, I, U)] = True          # at least one item per row ...
    dense[~nonempty] = False                                    # ... except the users without training items
    m = sp.csr_matrix(dense.astype(np.float32))
    m.sort_indices()
    return m


def _cases():
    """name -> (matrix, batch sizes).  Every matrix is used at worlds 2 and 3."""
    rng = np.random.default_rng(3)
    odd = rng.random(203) < 0.7                                  # 203 users: the last block is padded at both worlds
    big = rng.random(1501) < 0.85                                # > 1024 eligible users: the select path with distinct users
    tail = np.arange(90) < 45                                    # rows 45..89 empty: world 2 rank 1 / world 3 rank 2 hold none
    head = np.arange(91) < 29                                    # only rows 0..28: every batch lies in rank 0's block
    cases = {"odd": (_matrix(203, 57, odd, 0.08, 1), [1, 37, 1024]),
             "select": (_matrix(1501, 40, big, 0.05, 2), [1025, 1100]),
             "empty_rank": (_matrix(90, 33, tail, 0.1, 3), [16, 45, 50, 1030]),
             "one_block": (_matrix(91, 25, head, 0.1, 4), [8, 29, 1200])}
    n_sel = int(big.sum())
    cases["select"][1].append(n_sel)                             # a permutation through the select path
    n_odd = int(odd.sum())
    cases["odd"][1].extend([n_odd, n_odd + 3])                   # a permutation of the claim path, with replacement
    return cases


def block_rows(mat, part, rank):
    """The rank's training rows as ShardedDataset.train_rows() hands them out (padded CsrBlock, int32 global item ids)."""
    from mmssl_b200.dataset import CsrBlock
    from mmssl_b200.parallel import shard_rows_scipy
    lo, hi = part.bounds(rank)
    blk = shard_rows_scipy(mat, part, rank)
    return CsrBlock(blk.indptr.astype(np.int64), blk.indices.astype(np.int32), None, blk.shape, lo, hi)


def _batches_worker(rank, world, port, ret):
    _init(rank, world, port)
    try:
        from mmssl_b200.parallel import RowPartition
        from mmssl_b200.sampler import DeviceTripleSampler, ShardedTripleSampler
        errs = []
        for name, (mat, sizes) in _cases().items():
            pu = RowPartition(mat.shape[0], world)
            full = DeviceTripleSampler(mat, device="cpu", seed=SEED)
            mine = ShardedTripleSampler(block_rows(mat, pu, rank), pu, rank, device="cpu", seed=SEED)
            if mine.n_exist != full.exist.numel():
                errs.append(f"{name}: n_exist {mine.n_exist} vs {full.exist.numel()}")
            owned = mine.slot_hi - mine.slot_lo
            if name in ("empty_rank", "one_block") and rank == world - 1 and owned != 0:
                errs.append(f"{name}: the last rank owns {owned} slots")
            for b in sizes:
                for step in (0, 1, 6):
                    want = full.sample_into(torch.zeros(3, b, dtype=torch.int64), step=step)
                    step_dev = torch.full((1,), step, dtype=torch.int32) if step == 6 else None
                    got = mine.sample_into(torch.full((3, b), -1, dtype=torch.int64), step_dev=step_dev, step=0 if step_dev is not None else step)
                    if not torch.equal(got, want):
                        errs.append(f"{name}: B={b} step={step}: {(got != want).sum().item()} entries differ")
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_sampler_bitwise_equal_to_device_sampler(world):
    ret = mp.Manager().dict()
    mp.spawn(_batches_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert len(ret) == world
    for rank in range(world):
        assert ret[rank] == [], (rank, ret[rank])


def test_owned_range_is_checked():
    """The entry point refuses an owned slot range outside [0, n_exist) instead of reading past `exist`."""
    from mmssl_b200 import _lib
    from tests.cuemu import harness
    lib = harness.emu_lib()
    z = torch.zeros(8, dtype=torch.int64)
    for lo, hi in ((-1, 2), (3, 2), (0, 9)):
        rc = lib.mmssl_sample_triples_owned(_lib.ptr(z), _lib.ptr(z), _lib.ptr(z), lo, hi, 0, 8, 4, 2, 1, None, 0, _lib.ptr(z),
                                            _lib.ptr(z), _lib.ptr(z), _lib.ptr(z), None)
        assert rc != 0, (lo, hi)


def _chain_worker(rank, port, shard_dir, ret):
    world = 2
    _init(rank, world, port)
    try:
        from mmssl_b200.dataset import ReferenceDataset, ShardedDataset
        from mmssl_b200.sampler import DeviceTripleSampler, ShardedTripleSampler
        ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
        full = DeviceTripleSampler(ds.train_mat, device="cpu", seed=SEED)
        mine = ShardedTripleSampler.from_dataset(ShardedDataset.open(shard_dir, rank, world), device="cpu", seed=SEED)
        n = full.exist.numel()
        errs = []
        for b in (16, n, n + 7, 1100):
            for step in (0, 3):
                want = full.sample_into(torch.zeros(3, b, dtype=torch.int64), step=step)
                got = mine.sample_into(torch.zeros(3, b, dtype=torch.int64), step=step)
                if not torch.equal(got, want):
                    errs.append(f"B={b} step={step}")
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


def test_whole_chain_from_shards(tmp_path):
    """dataset_small -> write_shards -> per-rank ShardedDataset.train_rows -> ShardedTripleSampler at world 2: bitwise the
    one-GPU sampler on the dataset's train_mat."""
    from mmssl_b200.dataset import ReferenceDataset, write_shards
    write_shards(ReferenceDataset.load(os.path.join(GOLD, "dataset_small")), str(tmp_path))
    ret = mp.Manager().dict()
    mp.spawn(_chain_worker, args=(_free_port(), str(tmp_path), ret), nprocs=2, join=True)
    for rank in range(2):
        assert ret[rank] == [], (rank, ret[rank])


# ---------------------------------------------------------------- the sampler inside the row-sharded step
def _problem():
    from mmssl_b200.synthetic import csr_norm, make_bipartite
    U, I, d, B = 203, 131, 64, 48
    r = make_bipartite(U, I, 1500, seed=5).tocsr()
    r = sp.csr_matrix(r.multiply(np.arange(U)[:, None] % 7 != 3))     # users without training items in every block
    r.eliminate_zeros()
    r.sort_indices()
    g = torch.Generator().manual_seed(2)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, 40), "image_trans.bias": torch.randn(d, generator=g) * 0.1, "text_trans.weight": xav(d, 24),
         "text_trans.bias": torch.randn(d, generator=g) * 0.1, "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    feats = (torch.randn(I, 40, generator=g), torch.randn(I, 24, generator=g))
    masks = tuple(((torch.rand(I, d, generator=g) >= 0.2) / 0.8).float() for _ in range(2))
    return U, I, d, B, r, P, feats, masks


def _sharded(prob, rank, world, seed=SEED, sampled=True):
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem
    from mmssl_b200.sampler import ShardedTripleSampler
    from mmssl_b200.synthetic import csr_norm
    U, I, d, B, r, P, feats, masks = prob
    Pl, fl, gl, pu, pi = shard_problem(P, feats, csr_norm(r), csr_norm(r.T.tocsr()), rank, world, "cpu")
    smp = ShardedTripleSampler(block_rows(r, pu, rank), pu, rank, device="cpu", seed=seed) if sampled else None
    sh = RowShardedHotStep(Pl, fl, gl, HotStepConfig(embed_size=d, n_layers=2, batch_size=B, proj_impl="simt"), B, pu, pi, rank,
                           sampler=smp)
    sh.masks = tuple(pi.local(m, rank) for m in masks)
    return sh


def _step_worker(rank, port, ret):
    """World 2: two steps with the sampler against two steps fed the same batches by set_indices."""
    world = 2
    _init(rank, world, port)
    try:
        from mmssl_b200.engine import LIVE
        from mmssl_b200.sampler import DeviceTripleSampler
        prob = _problem()
        full = DeviceTripleSampler(prob[4], device="cpu", seed=SEED)
        sampled, fed = _sharded(prob, rank, world), _sharded(prob, rank, world, sampled=False)
        errs = []
        for step in range(2):
            out_s = sampled.run().clone()
            want = full.sample_into(torch.zeros(3, prob[3], dtype=torch.int64), step=step)
            if not torch.equal(sampled.idx, want):
                errs.append(f"step {step}: idx is not the one-GPU sampler's batch")
            fed.set_indices(*want)
            out_f = fed.run().clone()
            if not torch.equal(out_s, out_f):
                errs.append(f"step {step}: losses")
            for k in LIVE:
                if not (torch.equal(sampled.grads[k], fed.grads[k]) and torch.equal(sampled.P[k], fed.P[k])):
                    errs.append(f"step {step}: {k}")
        if sampled.meta().get("sampler_seed") != SEED or "sampler_seed" in fed.meta():
            errs.append("meta sampler_seed")
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


def test_rowshard_step_with_sampler_equals_set_indices():
    ret = mp.Manager().dict()
    mp.spawn(_step_worker, args=(_free_port(), ret), nprocs=2, join=True)
    for rank in range(2):
        assert ret[rank] == [], (rank, ret[rank])


def _save_worker(rank, port, directory, k, ret):
    """World 2: k sampled steps, save, then the batch the next step draws."""
    world = 2
    _init(rank, world, port)
    try:
        sh = _sharded(_problem(), rank, world)
        for _ in range(k):
            sh.run()
        sh.save(directory)
        sh.run()
        ret[rank] = sh.idx.clone()
    finally:
        dist.destroy_process_group()


def test_sampled_checkpoint_resumes_at_world1(monkeypatch, tmp_path):
    """Saved at world 2 after k sampled steps, read at world 1 into HotStep with DeviceTripleSampler of the same seed: its next
    batch is bitwise the world-2 run's.  Another seed is refused."""
    from mmssl_b200 import checkpoint
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import csr_norm
    from tests.cuemu import harness
    k, directory = 2, str(tmp_path / "w2")
    ret = mp.Manager().dict()
    mp.spawn(_save_worker, args=(_free_port(), directory, k, ret), nprocs=2, join=True)
    assert torch.equal(ret[0], ret[1])
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    U, I, d, B, r, P, feats, masks = _problem()
    full = checkpoint.read_sharded(directory, 1, 0)
    assert full["meta"]["sampler_seed"] == SEED
    g_ui, g_iu = BipartiteGraph.from_scipy(csr_norm(r), device="cpu"), BipartiteGraph.from_scipy(csr_norm(r.T.tocsr()), device="cpu")

    def hot(seed):
        hs = HotStep({k_: torch.zeros_like(v) for k_, v in P.items()}, tuple(FeatureStore(f.clone()) for f in feats), [g_ui, g_iu] * 3,
                     HotStepConfig(embed_size=d, n_layers=2, batch_size=B, proj_impl="simt"), batch=B,
                     sampler=DeviceTripleSampler(r, device="cpu", seed=seed))
        hs.engine.two_streams = False
        hs.masks = masks
        return hs

    hs = hot(SEED)
    hs.load_state_dict(full)
    assert int(hs.step_dev[0]) == k
    hs.run()
    assert torch.equal(hs.idx, ret[0])
    with pytest.raises(ValueError, match="sampler_seed"):
        hot(SEED + 1).load_state_dict(full)
