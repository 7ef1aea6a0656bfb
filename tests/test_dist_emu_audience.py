"""audience.ShardedAudience at world 2 and 3 over gloo, every rank running the real kernels under the cuemu emulator: each rank
ranks the listed items against its own user rows only, the partial lists travel by all_to_all_single to the ranks owning the
items, and the merged lists -- ``topk`` and the export read back with ``audience.read`` -- are bitwise the one-GPU ``Audience``'s
on the same tables.  The user count is not a multiple of the world size, one item list has no item of rank 0, and both exclusion
sets are covered.  At world 2 the whole row-sharded path of ``tools/recommend.py --audience`` (checkpoint load, the rank's final
tables, per-rank export) reads back the one-GPU lists on the gathered tables."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_dist_emu_sharded_eval import _MP, _free_port

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a):
    return np.ascontiguousarray(a.cpu().numpy() if torch.is_tensor(a) else a).view(np.uint8)


def _lists(world, rank, out_root, errs):
    from mmssl_b200 import audience
    from mmssl_b200.parallel import RowPartition
    from tests.test_gpu_zz_recommend import problem
    U, I, d, k = 61, 23, 8, 6
    assert U % world
    ua, ia, train = problem(U, I, d, 4, n_excl=(0, 9))
    rng = np.random.default_rng(4)
    test = {u: rng.choice(I, size=2, replace=False).tolist() for u in range(U)}
    val = {u: rng.choice(I, size=1, replace=False).tolist() for u in range(0, U, 3)}
    pu, pi = RowPartition(U, world), RowPartition(I, world)
    uc, ic = torch.from_numpy(ua), torch.from_numpy(ia)
    variants = {"shuffled": np.concatenate([rng.permutation(I), [0, I - 1, 0]]), "not_rank0": np.arange(pi.block, I)[::-1].copy(),
                "none": np.zeros(0, np.int64)}
    for exclude in ("train", "seen"):
        one = audience.Audience.from_rows(uc, train, test, val, I, k, exclude)
        sa = audience.ShardedAudience.from_rows(train, test, val, U, I, pu, pi, rank, k, exclude, device="cpu")
        for name, items in variants.items():
            out = os.path.join(out_root, f"w{world}_{exclude}_{name}")
            n = sa.export(pu.local(uc, rank), pi.local(ic, rank), items, out, chunk=4)
            if n != int((items // pi.block == rank).sum()):
                errs.append(f"{exclude}/{name}: {n} rows written")
            dist.barrier()
            q, i, s = audience.read(out)
            want_q = np.sort(items, kind="stable")
            wi, ws = one.topk(ic, want_q)
            if not (np.array_equal(q, want_q) and np.array_equal(i, wi.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))):
                errs.append(f"{exclude}/{name}: read-back lists differ from the one-GPU Audience")
            got_i, got_s, pos = sa.topk(pu.local(uc, rank), pi.local(ic, rank), items, chunk=5)
            wi, ws = one.topk(ic, items[pos])
            if not (torch.equal(got_i, wi) and np.array_equal(_bits(got_s), _bits(ws))):
                errs.append(f"{exclude}/{name}: topk differs")
            dist.barrier()


def _tool(rank, shard_dir, ckpt_dir, out_root, errs):
    """A RowShardedHotStep saved to a checkpoint; the tool's --sharded --audience export == the one-GPU Audience on the gathered
    final tables."""
    import importlib.util
    from mmssl_b200 import audience
    from mmssl_b200.dataset import ShardedDataset
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.parallel import all_gather_rows
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
    world = 2
    sh = ShardedDataset.open(shard_dir, rank, world)
    U, I, d, B, k = sh.n_users, sh.n_items, 32, 16, 5
    g = torch.Generator().manual_seed(4)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, sh.meta["image_dim"]), "image_trans.bias": torch.randn(d, generator=g) * 0.1,
         "text_trans.weight": xav(d, sh.meta["text_dim"]), "text_trans.bias": torch.randn(d, generator=g) * 0.1,
         "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    Pl, fl, gl, pu, pi = shard_problem_from_disk(shard_dir, P, rank, world, "cpu")
    st = RowShardedHotStep(Pl, fl, gl, HotStepConfig(embed_size=d, n_layers=2, batch_size=B), B, pu, pi, rank)
    st.save(ckpt_dir)
    u_f, i_f = st.final_embeddings()
    uf, itab = all_gather_rows(u_f, pu), all_gather_rows(i_f, pi)
    whole = ShardedDataset.open(shard_dir, 0, 1)
    spec = importlib.util.spec_from_file_location("recommend_tool", os.path.join(ROOT, "tools", "recommend.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    items = np.array([I - 1, 3, 0, 3, 20], np.int64)
    np.save(os.path.join(out_root, "items.npy"), items)
    for exclude in ("train", "seen"):
        out = os.path.join(out_root, f"tool_{exclude}")
        tool.main(["--sharded", ckpt_dir, "--shards", shard_dir, "--k", str(k), "--exclude", exclude, "--out", out, "--chunk", "2",
                   "--audience", "--items", os.path.join(out_root, "items.npy")])
        dist.barrier()
        q, i, s = audience.read(out)
        excl = audience.ShardedAudience.from_shards(whole, k, exclude, device="cpu").exclude
        wi, ws = audience.Audience(uf.contiguous(), excl, k).topk(itab.contiguous(), np.sort(items))
        if not (np.array_equal(q, np.sort(items)) and np.array_equal(i, wi.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))):
            errs.append(f"tool/{exclude}: the export differs from the one-GPU Audience")


def _worker(rank, world, port, shard_dir, ckpt_dir, out_root, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        torch.cuda.set_device = lambda d: None
        errs = []
        _lists(world, rank, out_root, errs)
        if shard_dir:
            _tool(rank, shard_dir, ckpt_dir, out_root, errs)
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_audience_bitwise_one_gpu(tmp_path, world):
    shard_dir = ckpt_dir = ""
    if world == 2:
        from mmssl_b200.dataset import ReferenceDataset, write_shards
        shard_dir, ckpt_dir = str(tmp_path / "shards"), str(tmp_path / "ckpt")
        write_shards(ReferenceDataset.load(os.path.join(GOLD, "dataset_small")), shard_dir)
    out_root = str(tmp_path / "out")
    os.makedirs(out_root)
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), shard_dir, ckpt_dir, out_root, ret), nprocs=world, join=True)
    for rank in range(world):
        assert ret[rank] == [], (rank, ret[rank])
