"""similar.ShardedSimilarItems at world 2 over gloo, every rank running the real kernels under the cuemu emulator, on
tests/golden/dataset_small (43 items: rank 1's block is padded).  A RowShardedHotStep saved to a checkpoint gives each rank its
block of every space -- ``final_embeddings`` for "model", ``projections`` for "image" / "text" -- and in every space ``topk`` and
the export read back with ``similar.read`` are bitwise the one-GPU ``SimilarItems`` lists: on the gathered final item table, and
on the one-GPU projection of the whole catalogue (the rank's projection is bitwise that projection's rows).  Then the whole
row-sharded path of tools/similar_items.py (load at world 2, the rank's table, per-rank export) reads back the same lists."""
import os

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_dist_emu_sharded_eval import _MP, _free_port

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a):
    return np.ascontiguousarray(a.cpu().numpy() if torch.is_tensor(a) else a).view(np.uint8)


def _worker(rank, port, shard_dir, ckpt_dir, out_root, ret):
    world = 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        torch.cuda.set_device = lambda d: None
        import importlib.util
        from mmssl_b200 import similar
        from mmssl_b200.dataset import ShardedDataset
        from mmssl_b200.engine import Engine, FeatureStore
        from mmssl_b200.hotstep import HotStepConfig
        from mmssl_b200.parallel import all_gather_rows
        from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
        sh = ShardedDataset.open(shard_dir, rank, world)
        U, I, d, B, k = sh.n_users, sh.n_items, 32, 16, 9
        g = torch.Generator().manual_seed(4)
        xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
        P = {"image_trans.weight": xav(d, sh.meta["image_dim"]), "image_trans.bias": torch.randn(d, generator=g) * 0.1,
             "text_trans.weight": xav(d, sh.meta["text_dim"]), "text_trans.bias": torch.randn(d, generator=g) * 0.1,
             "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d)}
        Pl, fl, gl, pu, pi = shard_problem_from_disk(shard_dir, P, rank, world, "cpu")
        assert I % 2 and pi.block * world > I
        st = RowShardedHotStep(Pl, fl, gl, HotStepConfig(embed_size=d, n_layers=2, batch_size=B), B, pu, pi, rank)
        st.save(ckpt_dir)
        whole = ShardedDataset.open(shard_dir, 0, 1)
        feats = tuple(FeatureStore(torch.from_numpy(np.ascontiguousarray(whole.features(w))).float()) for w in ("image", "text"))
        xv, xt = similar.project(Engine(d, 2), {kk: v for kk, v in P.items()}, feats)
        i_f = st.final_embeddings()[1]
        pv, pt = st.projections()
        blocks = {"model": i_f, "image": pv, "text": pt}
        full = {"model": all_gather_rows(i_f, pi), "image": xv, "text": xt}
        errs = []
        lo, hi = pi.bounds(rank)
        for space, blk in (("image", pv), ("text", pt)):
            if not np.array_equal(_bits(blk[:hi - lo].contiguous()), _bits(full[space][lo:hi].contiguous())):
                errs.append(f"{space}: the rank's projection differs from the one-GPU projection's rows")
        rng = np.random.default_rng(5)
        variants = {"shuffled": np.concatenate([rng.permutation(I), [0, I - 1, 0]]), "rank1_only": np.arange(pi.block, I)[::-1].copy()}
        for space in similar.SPACES:
            one = similar.SimilarItems(full[space], k, space)
            sr = similar.ShardedSimilarItems(pi, rank, k, space, device="cpu")
            for name, items in variants.items():
                out = os.path.join(out_root, f"{space}_{name}")
                n = sr.export(blocks[space], items, out, chunk=4)
                if n != int((items // pi.block == rank).sum()):
                    errs.append(f"{space}/{name}: {n} rows written")
                dist.barrier()
                q, i, s = similar.read(out)
                want_q = np.sort(items, kind="stable")
                wi, ws = one.topk(want_q)
                if not (np.array_equal(q, want_q) and np.array_equal(i, wi.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))):
                    errs.append(f"{space}/{name}: read-back lists differ from the one-GPU SimilarItems")
                got_i, got_s, pos = sr.topk(blocks[space], items)
                wi, ws = one.topk(items[pos])
                if not (torch.equal(got_i, wi) and np.array_equal(_bits(got_s), _bits(ws))):
                    errs.append(f"{space}/{name}: topk differs")
                dist.barrier()
        spec = importlib.util.spec_from_file_location("similar_tool", os.path.join(ROOT, "tools", "similar_items.py"))
        tool = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(tool)
        for space in similar.SPACES:
            out = os.path.join(out_root, f"tool_{space}")
            tool.main(["--sharded", ckpt_dir, "--shards", shard_dir, "--k", str(k), "--space", space, "--out", out, "--chunk", "7"])
            dist.barrier()
            q, i, s = similar.read(out)
            wi, ws = similar.SimilarItems(full[space], k, space).topk(np.arange(I))
            if not (np.array_equal(q, np.arange(I)) and np.array_equal(i, wi.numpy().astype(np.int32)) and np.array_equal(_bits(s), _bits(ws))):
                errs.append(f"tool/{space}: the export differs from the one-GPU SimilarItems")
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


def test_sharded_similar_bitwise_one_gpu(tmp_path):
    from mmssl_b200.dataset import ReferenceDataset, write_shards
    shard_dir, ckpt_dir = str(tmp_path / "shards"), str(tmp_path / "ckpt")
    write_shards(ReferenceDataset.load(os.path.join(GOLD, "dataset_small")), shard_dir)
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(port, shard_dir, ckpt_dir, str(tmp_path / "out"), ret), nprocs=2, join=True)
    for rank in range(2):
        assert ret[rank] == [], (rank, ret[rank])
