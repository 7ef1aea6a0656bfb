"""recommend.ShardedRecommender at world 2 over gloo, every rank running the real ranking kernels under the cuemu emulator: every
rank's export, read back with ``recommend.read``, is bitwise the one-GPU ``Recommender`` on the gathered tables, for both
exclusion sets, for a shuffled user list with repeats and for a list with no user in rank 0's block (no launch there).  Also the
whole row-sharded path of tools/recommend.py: write_shards -> RowShardedHotStep.save -> the tool (load at world 2, eval-mode
forward, ShardedRecommender.from_shards, per-rank export) -> read, bitwise the one-GPU lists on the gathered final embeddings."""
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


def _worker(rank, port, out_root, ret):
    world = 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        from mmssl_b200 import recommend
        from mmssl_b200.dataset import ReferenceDataset
        from mmssl_b200.parallel import RowPartition
        ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
        U, I = ds.train_mat.shape
        k, d = 12, 16
        g = torch.Generator().manual_seed(3)
        ua, ia = torch.randn(U, d, generator=g), torch.randn(I, d, generator=g)
        pu, pi = RowPartition(U, world), RowPartition(I, world)
        u_local, i_local = pu.local(ua, rank), pi.local(ia, rank)
        launches = [0]
        real = recommend.Recommender._launch

        def counted(self, *a):
            launches[0] += 1
            return real(self, *a)
        recommend.Recommender._launch = counted
        errs = []
        rng = np.random.default_rng(5)
        for exclude in ("train", "seen"):
            one = recommend.Recommender.from_rows(ia, ds.train_items, ds.test_set, ds.val_set, U, k, exclude)
            sr = recommend.ShardedRecommender.from_rows(ds.train_items, ds.test_set, ds.val_set, U, I, pu, pi, rank, k, exclude,
                                                        device="cpu")
            variants = {"shuffled": np.concatenate([rng.permutation(U), [0, U - 1, 0]]), "rank1_only": np.arange(pu.block, U)[::-1]}
            for name, users in variants.items():
                out = os.path.join(out_root, f"{exclude}_{name}")
                launches[0] = 0
                n = sr.export(u_local, i_local, users, out, chunk=9)
                if n != int((users // pu.block == rank).sum()):
                    errs.append(f"{exclude}/{name}: {n} rows written")
                if name == "rank1_only" and rank == 0 and launches[0]:
                    errs.append("rank 0 launched with no user of its block")
                dist.barrier()
                u, i, s = recommend.read(out)
                want_u = np.sort(users, kind="stable")
                wi, ws = one.topk(ua, want_u)
                if not (np.array_equal(u, want_u) and np.array_equal(i, wi.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))):
                    errs.append(f"{exclude}/{name}: read-back lists differ from the one-GPU Recommender")
                got_i, got_s, pos = sr.topk(u_local, i_local, users)
                wi, ws = one.topk(ua, users[pos])
                if not (torch.equal(got_i, wi) and np.array_equal(_bits(got_s), _bits(ws))):
                    errs.append(f"{exclude}/{name}: topk differs")
                dist.barrier()
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


def test_sharded_export_bitwise_one_gpu(tmp_path):
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(port, str(tmp_path), ret), nprocs=2, join=True)
    for rank in range(2):
        assert ret[rank] == [], (rank, ret[rank])


def _tool_worker(rank, port, shard_dir, ckpt_dir, out_root, ret):
    world = 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        torch.cuda.set_device = lambda d: None
        import importlib.util
        from mmssl_b200 import recommend
        from mmssl_b200.dataset import ShardedDataset
        from mmssl_b200.hotstep import HotStepConfig
        from mmssl_b200.parallel import all_gather_rows
        from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
        sh = ShardedDataset.open(shard_dir, rank, world)
        U, I, d, B = sh.n_users, sh.n_items, 64, 16
        g = torch.Generator().manual_seed(4)
        xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
        P = {"image_trans.weight": xav(d, sh.meta["image_dim"]), "image_trans.bias": torch.randn(d, generator=g) * 0.1,
             "text_trans.weight": xav(d, sh.meta["text_dim"]), "text_trans.bias": torch.randn(d, generator=g) * 0.1,
             "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d)}
        Pl, fl, gl, pu, pi = shard_problem_from_disk(shard_dir, P, rank, world, "cpu")
        st = RowShardedHotStep(Pl, fl, gl, HotStepConfig(embed_size=d, n_layers=2, batch_size=B), B, pu, pi, rank)
        st.save(ckpt_dir)
        u_f, i_f = st.final_embeddings()
        u_full, i_full = all_gather_rows(u_f, pu), all_gather_rows(i_f, pi)
        spec = importlib.util.spec_from_file_location("recommend_tool", os.path.join(ROOT, "tools", "recommend.py"))
        tool = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(tool)
        errs = []
        whole = ShardedDataset.open(shard_dir, 0, 1)
        pair = lambda b: (b.indptr, b.indices)
        for exclude in ("train", "seen"):
            out = os.path.join(out_root, exclude)
            tool.main(["--sharded", ckpt_dir, "--shards", shard_dir, "--k", "9", "--exclude", exclude, "--out", out, "--chunk", "7"])
            dist.barrier()
            rows = pair(whole.train_rows())
            if exclude == "seen":
                rows = recommend.union_csr(rows, pair(whole.held("val")), pair(whole.held("test")))
            one = recommend.Recommender(i_full, recommend._device_csr(*rows, "cpu"), 9)
            u, i, s = recommend.read(out)
            wi, ws = one.topk(u_full, np.arange(U))
            if not (np.array_equal(u, np.arange(U)) and np.array_equal(i, wi.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))):
                errs.append(f"{exclude}: the tool's export differs from the one-GPU Recommender")
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


def test_recommend_tool_row_sharded(tmp_path):
    from mmssl_b200.dataset import ReferenceDataset, write_shards
    shard_dir, ckpt_dir = str(tmp_path / "shards"), str(tmp_path / "ckpt")
    write_shards(ReferenceDataset.load(os.path.join(GOLD, "dataset_small")), shard_dir)
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_tool_worker, args=(port, shard_dir, ckpt_dir, str(tmp_path / "out"), ret), nprocs=2, join=True)
    for rank in range(2):
        assert ret[rank] == [], (rank, ret[rank])
