"""evaluate.ShardedEvaluator on the H100: at world 1 (one rank holds every block) on the golden cases and a Baby-size case in
both modes, result, per-user rows, AUC and ranked lists bitwise the Evaluator's; on 2 GPUs (skipped below 2) the whole path --
row-sharded eval-mode forward, item all-gather, ranking, row gather + reduce -- through tools/sharded_eval_bench.py `check`,
bitwise the one-GPU Evaluator's on the all-gathered tables.  The 2-rank path runs on the CPU emulator over gloo in
tests/test_dist_emu_sharded_eval.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_dist_emu_sharded_eval import FAMILIES, _rows, compare

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _world_one(train, test, val, U, I, Ks, flag):
    from mmssl_b200.evaluate import Evaluator, ShardedEvaluator
    from mmssl_b200.parallel import RowPartition
    ev = Evaluator(train, test, val, U, I, Ks, test_flag=flag)
    se = ShardedEvaluator.from_rows(train, test, val, U, I, RowPartition(U, 1), RowPartition(I, 1), 0, Ks, flag)
    return ev, se


@pytest.mark.parametrize("case", [c for f in sorted(FAMILIES) for c in FAMILIES[f]])
def test_world_one_golden_bitwise(case):
    g = np.load(os.path.join(GOLD, case + ".npz"))
    Ks = [int(k) for k in g["Ks"]]
    U, I = g["ua"].shape[0], g["ia"].shape[0]
    flag = "full" if "full" in case else "part"
    ev, se = _world_one(*[_rows(g[f"{s}_indptr"], g[f"{s}_indices"]) for s in ("train", "test", "val")], U, I, Ks, flag)
    ua, ia = torch.from_numpy(g["ua"]).cuda(), torch.from_numpy(g["ia"]).cuda()
    for split in ("test", "val"):
        users = g[f"{split}_users"].astype(np.int64)
        for us in (users, users[::-1].copy(), np.concatenate([users, users[:7]])):
            bad, _ = compare(ev, se, ua, ia, ua, ia, list(us), split == "val")
            assert bad == [], (split, bad)


@pytest.mark.parametrize("flag", ["part", "full"])
def test_world_one_baby_size_bitwise(flag):
    """Baby-sized tables (19445 x 7050, d = 64), 2048 users in shuffled order."""
    from mmssl_b200.synthetic import CONFIGS, make_bipartite
    U, I, nnz, d, *_ = CONFIGS["baby"]
    tr = make_bipartite(U, I, nnz, seed=3).tocsr()
    tr.sort_indices()
    rng = np.random.default_rng(2)
    held = {u: rng.choice(I, size=int(rng.integers(1, 9)), replace=False).tolist() for u in range(U)}
    train = {u: tr.indices[tr.indptr[u]:tr.indptr[u + 1]].tolist() for u in range(U) if tr.indptr[u + 1] > tr.indptr[u]}
    ua = torch.from_numpy(rng.standard_normal((U, d)).astype(np.float32)).cuda()
    ia = torch.from_numpy(rng.standard_normal((I, d)).astype(np.float32)).cuda()
    ev, se = _world_one(train, held, {}, U, I, [10, 20, 50], flag)
    bad, _ = compare(ev, se, ua, ia, ua, ia, rng.permutation(U)[:2048].tolist(), False)
    assert bad == [], bad


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_eval_two_gpus():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29546", os.path.join(ROOT, "tools", "sharded_eval_bench.py"), "tiktok", "check", "--iters", "1"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert res["n_gpus"] == 2 and res["check"] is True, res


def _state(obj, prefix="", seen=None, out=None):
    """Copies of every tensor reachable from a step object (its buffers, parameters, optimiser state, graph operands,
    feature stores, workspaces): what a replay of its captured graph can read."""
    seen = set() if seen is None else seen
    out = {} if out is None else out
    if id(obj) in seen:
        return out
    seen.add(id(obj))
    if torch.is_tensor(obj):
        out[prefix] = obj.detach().clone()
    elif isinstance(obj, dict):
        for k, v in obj.items():
            _state(v, f"{prefix}[{k}]", seen, out)
    elif isinstance(obj, (list, tuple)):
        for j, v in enumerate(obj):
            _state(v, f"{prefix}[{j}]", seen, out)
    elif type(obj).__module__.startswith("mmssl_b200") and hasattr(obj, "__dict__"):
        for k, v in vars(obj).items():
            _state(v, f"{prefix}.{k}", seen, out)
    return out


def test_eval_between_replays_of_captured_step():
    """World 1: an evaluation (eval-mode forward + ShardedEvaluator) between two replays of a captured row-sharded step leaves
    every tensor the step holds bitwise as it was (but the SpMM scratch partials), and the next replay's losses agree with a twin step that never evaluates
    (within the run-to-run spread of the step's reductions on the device)."""
    if not torch.cuda.is_available():
        pytest.skip("CUDA graph capture needs a device")
    from mmssl_b200.evaluate import ShardedEvaluator
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("tiny", seed=3)
    U, I, d, B = ds.n_users, ds.n_items, 64, 64
    g = torch.Generator().manual_seed(5)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, ds.dv), "image_trans.bias": torch.zeros(d), "text_trans.weight": xav(d, ds.dt),
         "text_trans.bias": torch.zeros(d), "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    feats = (torch.randn(I, ds.dv, generator=g), torch.randn(I, ds.dt, generator=g))
    masks = tuple((((torch.rand(I, d, generator=g) >= 0.1) / 0.9).float()).cuda() for _ in range(2))
    users, pos, neg = torch.randperm(U, generator=g)[:B], torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
    cfg = HotStepConfig(embed_size=d, n_layers=2, batch_size=B)
    steps = []
    for _ in range(2):
        Pl, fl, gl, pu, pi = shard_problem(P, feats, ds.ui_norm, ds.iu_norm, 0, 1, "cuda")
        st = RowShardedHotStep(Pl, fl, gl, cfg, B, pu, pi, 0)
        st.masks = masks
        st.set_indices(users, pos, neg)
        st.capture()
        steps.append(st)
    a, b = steps
    tr = ds.train.tocsr()
    held = {u: [int((u * 7) % I)] for u in range(U)}
    train = {u: tr.indices[tr.indptr[u]:tr.indptr[u + 1]].tolist() for u in range(U) if tr.indptr[u + 1] > tr.indptr[u]}
    se = ShardedEvaluator.from_rows(train, held, held, U, I, a.pu, a.pi, 0, [5, 10], "full")
    for s in range(4):
        if s == 2:
            torch.cuda.synchronize()
            before = _state(a)
            res = a.test(se, list(range(U)), False)
            torch.cuda.synchronize()
            after = _state(a)
            assert np.all(np.isfinite(res["recall"])) and len(before) > 50 and before.keys() == after.keys()
            for k, t in before.items():
                if "._work[" in k and k.endswith("][0]"):     # SpMM split-row partials: scratch every launch writes before reading
                    continue
                same = torch.equal(t, after[k]) if t.dtype == torch.bool else torch.equal(t.reshape(-1).view(torch.uint8), after[k].reshape(-1).view(torch.uint8))
                assert same, k
        oa, ob = a.replay().clone(), b.replay().clone()
        torch.cuda.synchronize()
        assert float(((oa - ob).abs() / ob.abs().clamp_min(1e-12)).max()) < 1e-5, (s, oa, ob)
