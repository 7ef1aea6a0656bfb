"""foldin.ShardedFoldIn at world 2 and 3 over gloo, every rank running the real kernels under the cuemu emulator, from a
RowShardedHotStep: each rank gathers the item-side tables once (``fold_tables``), folds and ranks the queries it is given -- id
queries of the users of its block, new-user queries -- and its lists are bitwise the one-GPU ``FoldIn``'s on the gathered tables,
for both exclusion sets.  The last user block is padded, one rank is given no query at all, and an id query of a user of another
rank is refused.  ``tools/recommend.py --sharded --fold-in`` from the step's checkpoint writes per-rank files that read back as
the one-GPU lists of every query of the file."""
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


def queries(U, I, n, seed):
    """(rows, users): n random rows, ids for about half of them (a spread over every user block), -1 for the rest."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 12, n)
    ip = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ix = rng.integers(0, I, int(ip[-1])).astype(np.int64)
    users = np.where(rng.random(n) < 0.5, rng.integers(0, U, n), -1).astype(np.int64)
    users[:2] = [0, U - 1]
    return (ip, ix), users


def _run(rank, world, shard_dir, ckpt_dir, out_root, errs):
    import importlib.util
    from mmssl_b200 import foldin
    from mmssl_b200.dataset import ShardedDataset
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.parallel import all_gather_rows
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
    sh = ShardedDataset.open(shard_dir, rank, world)
    U, I, d, B, k = sh.n_users, sh.n_items, 32, 16, 7
    g = torch.Generator().manual_seed(6)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, sh.meta["image_dim"]), "image_trans.bias": torch.randn(d, generator=g) * 0.1,
         "text_trans.weight": xav(d, sh.meta["text_dim"]), "text_trans.bias": torch.randn(d, generator=g) * 0.1,
         "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    Pl, fl, gl, pu, pi = shard_problem_from_disk(shard_dir, P, rank, world, "cpu")
    if U % world == 0:
        errs.append(f"{U} users fill every block of world {world}: no padded block")
    st = RowShardedHotStep(Pl, fl, gl, HotStepConfig(embed_size=d, n_layers=2, batch_size=B), B, pu, pi, rank)
    st.save(ckpt_dir)
    tables = st.fold_tables()
    fi = foldin.ShardedFoldIn.from_dataset(tables, sh, 0.55)
    gat = lambda t, p: all_gather_rows(t.detach().contiguous(), p)
    whole = ShardedDataset.open(shard_dir, 0, 1)
    pair = lambda b: (np.asarray(b.indptr, np.int64), np.asarray(b.indices, np.int64))
    held = (pair(whole.train_rows()), pair(whole.held("val")), pair(whole.held("test")))
    one = foldin.FoldIn(gat(tables["u0"], pu)[:U], [gat(t, pi)[:I] for t in tables["layers"]], gat(tables["xv"], pi)[:I],
                        gat(tables["xt"], pi)[:I], gat(tables["i_f"], pi)[:I], 0.55, held)
    rows, users = queries(U, I, 40, 3)
    lo, hi = pu.bounds(rank)
    for exclude in ("train", "seen"):
        for name in ("mine", "none"):
            pick = fi.mine(users) if name == "mine" else np.zeros(0, np.int64)
            if name == "mine" and rank == world - 1:
                pick = np.concatenate([pick, np.nonzero(users < 0)[0]])
            if name == "none" and rank != world - 1:      # the last rank is given nothing here
                pick = np.nonzero(users < 0)[0]
            q, us = foldin.take_rows(rows, pick), users[pick]
            got = fi.topk(q, k, us, exclude)
            want = one.topk(q, k, us, exclude)
            if not (torch.equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1]))):
                errs.append(f"{exclude}/{name}: rank {rank}'s lists differ from the one-GPU FoldIn")
    foreign = (lo + pu.block) % U
    try:
        fi.topk(foldin.take_rows(rows, np.array([0])), k, np.array([foreign]))
        errs.append(f"user {foreign} of another rank was not refused")
    except ValueError as e:
        if "not held by rank" not in str(e):
            errs.append(str(e))
    # the tool from the checkpoint
    spec = importlib.util.spec_from_file_location("recommend_tool", os.path.join(ROOT, "tools", "recommend.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    path = os.path.join(out_root, "queries.npz")
    if rank == 0:
        np.savez(path, indptr=rows[0], indices=rows[1], users=users)
    dist.barrier()
    for exclude in ("train", "seen"):
        out = os.path.join(out_root, f"tool_{exclude}")
        tool.main(["--sharded", ckpt_dir, "--shards", shard_dir, "--k", str(k), "--exclude", exclude, "--out", out, "--chunk", "3",
                   "--fold-in", path])
        dist.barrier()
        qn, i, s = foldin.read(out)
        wi, ws = one.topk(rows, k, users, exclude)
        if not (np.array_equal(qn, np.arange(users.size)) and np.array_equal(i, wi.numpy().astype(np.int32)) and
                np.array_equal(_bits(s), _bits(ws))):
            errs.append(f"tool/{exclude}: the export differs from the one-GPU FoldIn")


def _worker(rank, world, port, shard_dir, ckpt_dir, out_root, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        torch.cuda.set_device = lambda d: None
        errs = []
        _run(rank, world, shard_dir, ckpt_dir, out_root, errs)
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_foldin_bitwise_one_gpu(tmp_path, world):
    from mmssl_b200.dataset import ReferenceDataset, write_shards
    shard_dir, ckpt_dir = str(tmp_path / "shards"), str(tmp_path / "ckpt")
    write_shards(ReferenceDataset.load(os.path.join(GOLD, "dataset_small")), shard_dir)
    out_root = str(tmp_path / "out")
    os.makedirs(out_root)
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), shard_dir, ckpt_dir, out_root, ret), nprocs=world, join=True)
    for rank in range(world):
        assert ret[rank] == [], (rank, ret[rank])
