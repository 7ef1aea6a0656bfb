"""evaluate.ShardedEvaluator at world sizes 2 and 3 over gloo, every rank running the REAL evaluation kernels under the cuemu
emulator: on the golden cases (odd user / item counts, so the last blocks are padded), both splits, every rank's result, mean
AUC and per-user rows are bitwise those of the single-process Evaluator on the same tables, every ranked list is the one
Evaluator ranks at the same position, and the result matches the reference's golden vectors.  Also: users_to_test shuffled,
with duplicates, or all in one block (the other ranks hold none of them)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FAMILIES = {"part": ["eval_random", "eval_ties", "eval_short"],
            "full": ["eval_full_random", "eval_full_ties", "eval_full_short", "eval_full_edges"],
            "wide": ["eval_wide_random", "eval_wide_ties", "eval_wide_short", "eval_wide_full"]}
EXACT = {"eval_ties", "eval_full_ties", "eval_full_edges", "eval_wide_ties", "eval_wide_full"}   # scores exact in fp32


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class _MP:
    def setattr(self, o, n, v):
        setattr(o, n, v)


def _rows(indptr, indices):
    return {u: indices[indptr[u]:indptr[u + 1]].tolist() for u in range(len(indptr) - 1) if indptr[u + 1] > indptr[u]}


def _bits(t):
    return np.ascontiguousarray(t.cpu().numpy()).view(np.uint8)


def _auc_bound(g, split, users, auc_golden):
    """|mean AUC - reference| allowed when fp32 scores summed in another order reorder the one closest pair of a user:
    the mean over users of 1 / (|P| |N|) (tests/test_gpu_zz_eval_full.py, per user)."""
    tp, ti, hp, hi = g["train_indptr"], g["train_indices"], g[f"{split}_indptr"], g[f"{split}_indices"]
    I = g["ia"].shape[0]
    b = []
    for k, u in enumerate(users):
        if np.isnan(auc_golden[k]):
            continue
        cand = np.setdiff1d(np.arange(I), ti[tp[u]:tp[u + 1]])
        P = int(np.isin(cand, hi[hp[u]:hp[u + 1]]).sum())
        b.append(1.0 / (P * (len(cand) - P)))
    return float(np.sum(b)) / max(len(users), 1) + 1e-12


def compare(ev, sh, ua, ia, u_local, i_local, users, is_val):
    """Bitwise: result, per_user, AUC, and the rank's ranked / ranked_scores / hits rows against Evaluator's at the same
    positions; test_torch dicts equal.  Returns a list of mismatch descriptions."""
    bad = []
    want = ev.rank(ua, ia, users, is_val)
    got = sh.rank(u_local, i_local, users, is_val)
    keys = ("result", "per_user") + (("auc",) if ev.test_flag == "full" else ())
    for k in keys:
        if got[k].shape != want[k].shape or not np.array_equal(_bits(got[k]), _bits(want[k])):
            bad.append(k)
    pos = got["positions"].numpy()
    for k in ("ranked", "ranked_scores", "hits"):
        if not np.array_equal(_bits(got[k]), _bits(want[k][torch.from_numpy(pos)])):
            bad.append(k)
    rw, rg = ev.test_torch(ua, ia, users, is_val), sh.test_torch(u_local, i_local, users, is_val)
    for k in ("precision", "recall", "ndcg", "hit_ratio"):
        if not np.array_equal(rw[k].view(np.uint64), rg[k].view(np.uint64)):
            bad.append("test_torch/" + k)
    if not np.array_equal(np.float64(rw["auc"]), np.float64(rg["auc"]), equal_nan=True):
        bad.append("test_torch/auc")
    return bad, rg


def _worker(rank, world, port, family, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        from mmssl_b200.evaluate import Evaluator, ShardedEvaluator
        from mmssl_b200.parallel import RowPartition
        errs = []
        for case in FAMILIES[family]:
            g = np.load(os.path.join(GOLD, case + ".npz"))
            Ks = [int(k) for k in g["Ks"]]
            U, I = g["ua"].shape[0], g["ia"].shape[0]
            flag = "full" if "full" in case else "part"
            pu, pi = RowPartition(U, world), RowPartition(I, world)
            rows = [_rows(g[f"{s}_indptr"], g[f"{s}_indices"]) for s in ("train", "test", "val")]
            ev = Evaluator(*rows, U, I, Ks, device="cpu", test_flag=flag)
            sh = ShardedEvaluator.from_rows(*rows, U, I, pu, pi, rank, Ks, flag, device="cpu")
            ua, ia = torch.from_numpy(g["ua"]), torch.from_numpy(g["ia"])
            u_local, i_local = pu.local(ua, rank), pi.local(ia, rank)
            rng = np.random.default_rng(7)
            for split in ("test", "val"):
                users = g[f"{split}_users"].astype(np.int64)
                is_val = split == "val"
                first = users[users < pu.block]                     # all in rank 0's block: the other ranks hold none
                variants = {"golden": users, "shuffled": rng.permutation(users),
                            "duplicates": np.concatenate([users, users[::3], users[:5]]), "one_block": first}
                for name, us in variants.items():
                    bad, res = compare(ev, sh, ua, ia, u_local, i_local, list(us), is_val)
                    errs += [f"{case}/{split}/{name}: {b}" for b in bad]
                    if name != "golden":
                        continue
                    got = np.stack([res[k] for k in ("precision", "recall", "ndcg", "hit_ratio")])
                    tol = 1e-12 if case in EXACT else 2e-2               # fp32 summation order may swap near-ties
                    if not np.allclose(got, g[f"{split}_result"], rtol=0, atol=tol):
                        errs.append(f"{case}/{split}: result vs golden")
                    if flag == "full":
                        want = float(g[f"{split}_result_auc"])
                        tol = 1e-12 if case in EXACT else _auc_bound(g, split, users, g[f"{split}_auc_per_user"])
                        if not ((np.isnan(want) and np.isnan(res["auc"])) or abs(res["auc"] - want) <= tol):
                            errs.append(f"{case}/{split}: auc {res['auc']} vs golden {want}")
            try:
                sh.rank(u_local, i_local, [0, U], False)
                errs.append(f"{case}: an id >= n_users was accepted")
            except ValueError:
                pass
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_evaluator_bitwise_equal_to_evaluator(world, family):
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, family, ret), nprocs=world, join=True)
    assert len(ret) == world
    for rank in range(world):
        assert ret[rank] == [], (rank, ret[rank])


def _chain_worker(rank, port, shard_dir, schedule, ret):
    """write_shards -> ShardedDataset -> RowShardedHotStep.final_embeddings -> ShardedEvaluator.from_shards at world 2."""
    world = 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(_MP())
        from mmssl_b200.dataset import ReferenceDataset, ShardedDataset
        from mmssl_b200.engine import LIVE, FeatureStore
        from mmssl_b200.evaluate import Evaluator, ShardedEvaluator
        from mmssl_b200.graph import BipartiteGraph
        from mmssl_b200.hotstep import HotStep, HotStepConfig
        from mmssl_b200.parallel import all_gather_rows
        from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem_from_disk
        from mmssl_b200.synthetic import csr_norm
        from tests.golden_util import rel_err
        ds = ReferenceDataset.load(os.path.join(GOLD, "dataset_small"))
        R = ds.train_mat.astype(np.float32).tocsr()
        R.sort_indices()
        U, I = R.shape
        d, B, Ks = 64, 16, [2, 5, 10]
        g = torch.Generator().manual_seed(4)
        xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
        P = {"image_trans.weight": xav(d, ds.image_feats.shape[1]), "image_trans.bias": torch.randn(d, generator=g) * 0.1,
             "text_trans.weight": xav(d, ds.text_feats.shape[1]), "text_trans.bias": torch.randn(d, generator=g) * 0.1,
             "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d), "weight_dict.w_self_attention_cat": xav(4 * d, d)}
        users = torch.randperm(U, generator=g)[:B]
        pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
        cfg = HotStepConfig(embed_size=d, n_layers=2, batch_size=B, drop_rate=0.1, proj_impl="simt")
        errs = {}

        def step():
            Pl, fl, gl, pu, pi = shard_problem_from_disk(shard_dir, P, rank, world, "cpu")
            st = RowShardedHotStep(Pl, fl, gl, cfg, B, pu, pi, rank, schedule=schedule)
            st.set_indices(users, pos, neg)
            return st

        torch.manual_seed(11)
        st = step()
        u_f, i_f = st.final_embeddings()
        # ---- the eval-mode embeddings against the one-GPU eval-mode forward (the 1e-4 contract of the sharded step)
        u_full, i_full = all_gather_rows(u_f, st.pu), all_gather_rows(i_f, st.pi)
        g_ui, g_iu = BipartiteGraph.from_scipy(csr_norm(R), device="cpu"), BipartiteGraph.from_scipy(csr_norm(R.T.tocsr()), device="cpu")
        feats = (torch.from_numpy(np.asarray(ds.image_feats, np.float32)), torch.from_numpy(np.asarray(ds.text_feats, np.float32)))
        hs = HotStep({k: v.clone() for k, v in P.items()}, tuple(FeatureStore(f.clone()) for f in feats),
                     [g_ui, g_iu, g_ui, g_iu, g_ui, g_iu], cfg, batch=B)
        hs.engine.two_streams = False
        outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, None, want_sumsq=False)
        errs["u_f"], errs["i_f"] = rel_err(u_full, outs[0]), rel_err(i_full, outs[1])
        # ---- the evaluation: bitwise Evaluator on the all-gathered tables
        train = {u: R.indices[R.indptr[u]:R.indptr[u + 1]].tolist() for u in range(U) if R.indptr[u + 1] > R.indptr[u]}
        bad = []
        for flag in ("part", "full"):
            ev = Evaluator(train, ds.test_set, ds.val_set, U, I, Ks, device="cpu", test_flag=flag)
            se = ShardedEvaluator.from_shards(ShardedDataset.open(shard_dir, rank, world), Ks, flag, device="cpu")
            for is_val, rows in ((False, ds.test_set), (True, ds.val_set)):
                order = sorted(rows)
                b, res = compare(ev, se, u_full, i_full, u_f, i_f, order, is_val)
                bad += [f"{flag}/{is_val}: {x}" for x in b]
                via_step = st.test(se, order, is_val)
                for k in ("precision", "recall", "ndcg", "hit_ratio"):
                    if not np.array_equal(via_step[k], res[k]):
                        bad.append(f"{flag}/{is_val}: step.test {k}")
        errs["eval"] = bad
        # ---- one training step after the evaluations is bitwise the step without them (same RNG state for the dropout masks)
        out_eval = st.run().clone()
        p_eval = {k: st.P[k].clone() for k in LIVE}
        torch.manual_seed(11)
        plain = step()
        out_plain = plain.run().clone()
        errs["step_after_eval"] = not (torch.equal(out_eval, out_plain) and all(torch.equal(p_eval[k], plain.P[k]) for k in LIVE))
        ret[rank] = errs
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("schedule", ["reduce_scatter", "allgather"])
def test_whole_chain_from_shards(tmp_path, schedule):
    """dataset_small -> write_shards -> per-rank ShardedDataset -> RowShardedHotStep.final_embeddings ->
    ShardedEvaluator.from_shards at world 2: the evaluation is bitwise Evaluator's on the all-gathered embeddings, the
    embeddings are the one-GPU eval-mode forward's within 1e-4, and an evaluation leaves the next training step bitwise as is."""
    from mmssl_b200.dataset import ReferenceDataset, write_shards
    write_shards(ReferenceDataset.load(os.path.join(GOLD, "dataset_small")), str(tmp_path))
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_chain_worker, args=(port, str(tmp_path), schedule, ret), nprocs=2, join=True)
    for rank in range(2):
        e = dict(ret[rank])
        assert e["step_after_eval"] is False, (rank, e)
        assert e["u_f"] < 1e-4 and e["i_f"] < 1e-4, (rank, e)
        assert e["eval"] == [], (rank, e["eval"])
