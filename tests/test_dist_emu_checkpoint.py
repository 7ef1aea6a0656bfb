"""Row-sharded checkpoints that reshard (mmssl_b200/checkpoint.py: save_sharded / read_sharded), two gloo ranks running the
real kernel sources under the cuemu emulator.  World 2 -> world 1 and world 1 -> world 2 on odd row counts, so the row blocks
change and the last block is padded: the reassembled tables and moments are bitwise the saved rows with zero padding, and the
next step agrees with the continued run at the saving world size within the multi-GPU parity bound (1e-4, DESIGN section 2)."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

WORLD = 2
TOL = 1e-4


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class _MP:
    def setattr(self, o, n, v):
        setattr(o, n, v)


def _problem():
    from mmssl_b200.synthetic import csr_norm, make_bipartite
    U, I, d, B = 203, 131, 64, 48
    r = make_bipartite(U, I, 1500, seed=5)
    g = torch.Generator().manual_seed(2)
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    P = {"image_trans.weight": xav(d, 40), "image_trans.bias": torch.randn(d, generator=g) * 0.1, "text_trans.weight": xav(d, 24),
         "text_trans.bias": torch.randn(d, generator=g) * 0.1, "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d)}
    feats = (torch.randn(I, 40, generator=g), torch.randn(I, 24, generator=g))
    masks = tuple(((torch.rand(I, d, generator=g) >= 0.2) / 0.8).float() for _ in range(2))
    batches = [(torch.randperm(U, generator=g)[:B], torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g))
               for _ in range(2)]
    return U, I, d, B, csr_norm(r), csr_norm(r.T.tocsr()), P, feats, masks, batches


def _sharded(prob, rank, world, P=None):
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem
    U, I, d, B, a_ui, a_iu, P0, feats, masks, _ = prob
    Pl, fl, gl, pu, pi = shard_problem(P or P0, feats, a_ui, a_iu, rank, world, "cpu")
    sh = RowShardedHotStep(Pl, fl, gl, HotStepConfig(embed_size=d, n_layers=2, batch_size=B, proj_impl="simt"), B, pu, pi, rank)
    sh.masks = tuple(pi.local(m, rank) for m in masks)
    return sh


def _full_rows(sh, t, space):
    """The rank's real rows of a table as (lo, rows)."""
    part = sh.pu if space == "user" else sh.pi
    lo, hi = part.bounds(sh.rank)
    return lo, t[:hi - lo].clone()


def _step_result(sh):
    from mmssl_b200.engine import P_EI, P_EU
    out = sh.run().clone()
    g = {k: v.clone() for k, v in sh.grads.items()}
    g[P_EU] = _full_rows(sh, sh.grads[P_EU], "user")
    g[P_EI] = _full_rows(sh, sh.grads[P_EI], "item")
    return out, g


def _init(rank, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    from tests.cuemu import harness
    harness.set_order("fwd")
    harness.emulated_device(_MP())


def _save_worker(rank, port, directory, ret):
    """World 2: one step, save, then the continued step."""
    _init(rank, port)
    try:
        prob = _problem()
        sh = _sharded(prob, rank, WORLD)
        sh.set_indices(*prob[-1][0])
        sh.run()
        sh.save(directory)
        sh.set_indices(*prob[-1][1])
        ret[rank] = _step_result(sh)
    finally:
        dist.destroy_process_group()


def _load_worker(rank, port, directory, ret):
    """World 2: load a world-1 checkpoint into steps built on other parameters, then one step."""
    _init(rank, port)
    try:
        from mmssl_b200 import checkpoint
        from mmssl_b200.engine import LIVE, P_EI, P_EU
        prob = _problem()
        sh = _sharded(prob, rank, WORLD, P={k: torch.zeros_like(v) for k, v in prob[6].items()})
        sh.load(directory)
        ck = checkpoint.load(checkpoint.committed_files(directory)[0])
        exact = True
        for k, space in ((P_EU, "user"), (P_EI, "item")):
            part = sh.pu if space == "user" else sh.pi
            lo, hi = part.bounds(rank)
            for live, saved in ((sh.P[k], ck["model"][k]), (sh.m[k], ck["optim"]["m"][k]), (sh.v[k], ck["optim"]["v"][k])):
                exact &= bool(torch.equal(live[:hi - lo], saved[lo:hi])) and bool((live[hi - lo:] == 0).all())
        for k in LIVE:
            if k not in (P_EU, P_EI):
                exact &= bool(torch.equal(sh.P[k], ck["model"][k])) and bool(torch.equal(sh.m[k], ck["optim"]["m"][k]))
        exact &= int(sh.step_dev[0]) == 1
        sh.set_indices(*prob[-1][1])
        padding = (sh.pu.block * WORLD - sh.pu.n, sh.pi.block * WORLD - sh.pi.n)
        ret[rank] = (exact, padding, _step_result(sh))
    finally:
        dist.destroy_process_group()


def _compare(got, want):
    """got / want: (out5, grads with (lo, rows) for the tables) -> max relative error over losses and gradients."""
    from mmssl_b200.engine import P_EI, P_EU
    from tests.golden_util import rel_err
    out_g, g_g = got
    out_w, g_w = want
    errs = [float(((out_g - out_w).abs() / out_w.abs().clamp_min(1e-12)).max())]
    for k in g_g:
        if k in (P_EU, P_EI):
            (lo_g, rows_g), (lo_w, rows_w) = g_g[k], g_w[k]
            errs.append(rel_err(rows_g, rows_w[lo_g - lo_w:lo_g - lo_w + rows_g.shape[0]]))
        else:
            errs.append(rel_err(g_g[k], g_w[k]))
    return max(errs)


def test_world2_checkpoint_loads_at_world1(monkeypatch, tmp_path):
    from mmssl_b200 import checkpoint
    from mmssl_b200.engine import LIVE, P_EI, P_EU
    from tests.cuemu import harness
    directory = str(tmp_path / "w2")
    ret = mp.Manager().dict()
    mp.spawn(_save_worker, args=(_free_port(), directory, ret), nprocs=WORLD, join=True)
    paths = checkpoint.committed_files(directory)
    assert [os.path.basename(f) for f in paths] == ["rank00000-of-00002.ckpt", "rank00001-of-00002.ckpt"]
    assert sorted(os.listdir(directory)) == sorted([checkpoint.MANIFEST, os.path.basename(os.path.dirname(paths[0]))])
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    prob = _problem()
    U, I = prob[0], prob[1]
    full = checkpoint.read_sharded(directory, 1, 0)
    assert full["kind"] == "hotstep"
    files = [checkpoint.load(f) for f in paths]
    for k, space, n in ((P_EU, "user", U), (P_EI, "item", I)):
        for src, dst in ((lambda f: f["model"][k], full["model"][k]), (lambda f: f["optim"]["m"][k], full["optim"]["m"][k]),
                         (lambda f: f["optim"]["v"][k], full["optim"]["v"][k])):
            assert dst.shape[0] == n and torch.equal(torch.cat([src(f) for f in files]), dst), k
    # world 1 = the plain fused HotStep, which takes the reassembled state as it is
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    _, _, d, B, a_ui, a_iu, P, feats, masks, batches = prob
    g_ui, g_iu = BipartiteGraph.from_scipy(a_ui, device="cpu"), BipartiteGraph.from_scipy(a_iu, device="cpu")
    hs = HotStep({k: torch.zeros_like(v) for k, v in P.items()}, tuple(FeatureStore(f.clone()) for f in feats), [g_ui, g_iu] * 3,
                 HotStepConfig(embed_size=d, n_layers=2, batch_size=B, proj_impl="simt"), batch=B)
    hs.engine.two_streams = False
    hs.masks = masks
    hs.load_state_dict(full)
    assert int(hs.step_dev[0]) == 1
    hs.set_indices(*batches[1])
    out = hs.run().clone()
    got = (out, {k: ((0, hs.grads[k].clone()) if k in (P_EU, P_EI) else hs.grads[k].clone()) for k in LIVE})
    for rank in range(WORLD):
        out_w, g_w = ret[rank]
        # the world-2 rank's rows against the same rows of the world-1 step
        assert _compare((out_w, g_w), got) < TOL, rank


def test_world1_checkpoint_loads_at_world2(monkeypatch, tmp_path):
    from mmssl_b200 import checkpoint
    from tests.cuemu import harness
    directory = str(tmp_path / "w1")
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    prob = _problem()
    sh = _sharded(prob, 0, 1)
    sh.set_indices(*prob[-1][0])
    sh.run()
    sh.save(directory)
    assert [os.path.basename(f) for f in checkpoint.committed_files(directory)] == ["rank00000-of-00001.ckpt"]
    sh.set_indices(*prob[-1][1])
    want = _step_result(sh)
    monkeypatch.undo()
    ret = mp.Manager().dict()
    mp.spawn(_load_worker, args=(_free_port(), directory, ret), nprocs=WORLD, join=True)
    for rank in range(WORLD):
        exact, pad, got = ret[rank]
        assert exact, rank
        assert pad == (1, 1)                          # 203 and 131 rows over two ranks: the last block of each table is padded
        assert _compare(got, want) < TOL, rank
