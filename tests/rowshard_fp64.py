"""Float64 yardstick of the row-sharded hot step (``mmssl_b200.rowshard_step.RowShardedHotStep``), one rank of a world at a
time; shared by tests/test_dist_emu_rowshard_fp64.py (gloo ranks under the cuemu emulator) and tests/test_gpu_zz_rowshard_fp64.py
(world 1 in process; worlds 2 and 3 launched as ``python -m torch.distributed.run ... -m tests.rowshard_fp64``).  A helper, not
a test file: it extends tests/hotstep_fp64.py (problem, oracle, measures, floors, ledger) to a sharded step.

Ranks produce, the parent judges.  ``run_cases`` runs on every rank and returns, per case and optimiser step, numpy copies of
the five losses, the rank's padded row blocks of the two table gradients, the replicated gradients, ``P`` / ``m`` / ``v``
before and after the step and the batch rows ``self.rows``.  ``judge`` assembles the full tables from the ranks' blocks,
evaluates the oracle in float64 and float32 at the parameters the ranks held before each step (hotstep_fp64.reference) and
applies hotstep_fp64's measures -- so failures read like the hot step's -- with two more classes of rows:

  block edge                 the first and last real row of every rank's block
  split / heavy (rank operand)  item rows classed by their degree in the column-block operand a rank multiplies under the
                             "reduce_scatter" schedule (A[:, users_r]: split differently from the whole graph)

and exact invariants, no tolerance: padded rows of both table gradients are 0; padded rows of P, m and v are bitwise unchanged
by every optimiser step; the losses, ``self.rows``, the replicated gradients and the replicated parameters after each step are
bitwise equal on every rank.  The AdamW update of every tensor is checked from the device's own gradient
(test_gpu_zz_hotstep_fp64.assert_update).
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, replace
from typing import Dict, List, Optional, Tuple

import numpy as np
import scipy.sparse as sp
import torch

from tests import hotstep_fp64 as H

REPLICATED = tuple(k for k in H.LIVE if k not in (H.P_EU, H.P_EI))
KINDS = ("plain", "block edges", "one rank", "repeated", "no edge")


@dataclass(frozen=True)
class Case:
    """One sharded problem and how it is stepped.  ``terms``: HotStepConfig overrides (test_gpu_zz_hotstep_fp64.term_configs);
    ``kind``: the batch of every step (KINDS); ``steps`` optimiser steps, each with another batch and other masks."""
    U: int = 61
    I: int = 43
    d: int = 32
    B: int = 24
    K: int = 2
    heads: int = 4
    modal: str = "alias"
    route: str = "simt/simt"
    schedule: str = "reduce_scatter"
    kind: str = "plain"
    steps: int = 1
    drop: float = 0.2
    terms: Tuple[Tuple[str, float], ...] = ()
    dv: int = 24
    dt: int = 20
    seed: int = 0
    cuts: Tuple[int, int, int, int] = H.DEFAULT_CUTS
    train: Optional[str] = None             # synthetic.CONFIGS name: a full-size interaction graph

    @property
    def name(self) -> str:
        t = ",".join(f"{k}={v:g}" for k, v in self.terms)
        return (f"U={self.U} I={self.I} d={self.d} B={self.B} K={self.K} H={self.heads} {self.modal} {self.route} {self.schedule} "
                f"{self.kind} steps={self.steps} drop={self.drop:g}{' ' + t if t else ''}")


def config(c: Case):
    from mmssl_b200.hotstep import HotStepConfig
    return HotStepConfig(embed_size=c.d, n_layers=c.K, batch_size=c.B, head_num=c.heads, drop_rate=c.drop,
                         proj_impl=c.route.split("/")[0], **dict(c.terms))


def case_problem(c: Case) -> H.Problem:
    train = None
    if c.train is not None:
        from mmssl_b200.synthetic import CONFIGS, make_bipartite
        U, I, nnz = CONFIGS[c.train][:3]
        assert (U, I) == (c.U, c.I)
        train = make_bipartite(U, I, nnz, seed=c.seed)
    elif 12 * c.U > c.U * c.I:              # too few cells for train_matrix's 6 U distinct edges: half the cells, one bare user / item
        rng = np.random.default_rng(c.seed)
        R = rng.random((c.U, c.I)) < 0.5
        R[np.arange(c.U), rng.integers(0, c.I, c.U)] = True
        R[c.U - 2, :] = False
        R[:, c.I - 2] = False
        train = sp.csr_matrix(R.astype(np.float32))
    return H.problem(c.U, c.I, d=c.d, B=c.B, modal=c.modal, dv=c.dv, dt=c.dt, head_num=c.heads, seed=c.seed, cuts=c.cuts,
                     drop=c.drop, train=train)


def _parts(c: Case, world: int):
    from mmssl_b200.parallel import RowPartition
    return RowPartition(c.U, world), RowPartition(c.I, world)


def batches(c: Case, p: H.Problem, world: int) -> List[tuple]:
    """(users, pos, neg, masks) of every step: the problem's batch first, then fresh draws; `c.kind` edits every one."""
    from mmssl_b200.synthetic import TripleSampler
    pu, pi = _parts(c, world)
    draw = TripleSampler(p.train, seed=c.seed + 29)
    gen = torch.Generator().manual_seed(c.seed + 41)
    out = []
    for s in range(c.steps):
        u, po, ne = ((p.users.numpy(), p.pos.numpy(), p.neg.numpy()) if s == 0 else draw.sample(c.B))
        u, po, ne = (np.array(x, dtype=np.int64) for x in (u, po, ne))
        masks = p.masks if s == 0 else H.new_masks(c.I, c.d, c.drop, gen)
        rng = np.random.default_rng(c.seed + 101 * s)
        B = c.B
        if c.kind == "block edges":         # every rank's first and last real row, and the row just past its block
            eu = sorted({x for r in range(world) for x in (pu.bounds(r)[0], pu.bounds(r)[1] - 1, pu.bounds(r)[1])
                         if 0 <= x < c.U and pu.bounds(r)[1] > pu.bounds(r)[0]})
            ei = sorted({x for r in range(world) for x in (pi.bounds(r)[0], pi.bounds(r)[1] - 1, pi.bounds(r)[1])
                         if 0 <= x < c.I and pi.bounds(r)[1] > pi.bounds(r)[0]})
            assert len(eu) <= B and len(ei) <= B, (eu, ei, B)
            u[:len(eu)] = eu
            po[:len(ei)] = ei
            ne[B - len(ei):] = ei[::-1]
        elif c.kind == "one rank":          # the batch lies in the last rank's blocks: every other rank contributes only zeros
            ru = max(r for r in range(world) if pu.bounds(r)[1] > pu.bounds(r)[0])
            ri = max(r for r in range(world) if pi.bounds(r)[1] > pi.bounds(r)[0])
            (ulo, uhi), (ilo, ihi) = pu.bounds(ru), pi.bounds(ri)
            u, po, ne = rng.integers(ulo, uhi, B), rng.integers(ilo, ihi, B), rng.integers(ilo, ihi, B)
        elif c.kind == "repeated":          # repeated users, pos == neg, an item both positive and negative
            u[B // 2:] = u[:B - B // 2]
            u[1] = u[0]
            ne[::3] = po[::3]
            ne[1] = po[0]
        elif c.kind == "no edge":           # rows without an edge (train_matrix leaves user U - 2 and item I - 2 bare)
            u[0], po[min(1, B - 1)], ne[min(2, B - 1)] = c.U - 2, c.I - 2, c.I - 2
        out.append((u, po, ne, masks))
    return out


# ---------------------------------------------------------------------------------------------------------------- one rank
def _scipy(g) -> sp.csr_matrix:
    r, c, v, shape = g
    return sp.coo_matrix((v, (r, c)), shape=shape).tocsr()       # duplicates summed: the halves of hotstep_fp64 add up exactly


def shard_problem(p: H.Problem, cfg, rank: int, world: int, device, schedule="reduce_scatter", exchange="nccl",
                  optimizer_step=True, nce="simt", sampler=None, group=None):
    """The RowShardedHotStep of rank `rank` on problem `p`: the "distinct" and "empty" modality graphs become
    RowBlockGraph.from_scipy, aliased graphs stay the same objects, masks go in through RowPartition.local; projection route
    from cfg.proj_impl, InfoNCE route `nce`."""
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.rowshard_step import RowBlockGraph, RowShardedHotStep
    pu, pi = RowPartition(p.U, world), RowPartition(p.I, world)
    P = {k: p.params[k].to(device).clone().contiguous() for k in REPLICATED}
    P[H.P_EU] = pu.local(p.params[H.P_EU], rank).to(device).contiguous()
    P[H.P_EI] = pi.local(p.params[H.P_EI], rank).to(device).contiguous()
    feats = tuple(FeatureStore(pi.local(f, rank).to(device).contiguous(), keep_fp32=True) for f in p.feats)
    made = {}
    graphs = []
    for g in p.coo:
        if id(g) not in made:
            rows_u = g[3] == (p.U, p.I)
            made[id(g)] = RowBlockGraph.from_scipy(_scipy(g), pu if rows_u else pi, pi if rows_u else pu, rank, device)
        graphs.append(made[id(g)])
    with H.nce_route(nce):
        sh = RowShardedHotStep(P, feats, graphs, cfg, int(p.users.numel()), pu, pi, rank, group=group, optimizer_step=optimizer_step,
                               exchange=exchange, schedule=schedule, sampler=sampler)
    sh.masks = tuple(pi.local(m, rank).to(device).contiguous() for m in p.masks)
    sh.set_indices(p.users, p.pos, p.neg)
    return sh


def snapshot(sh) -> dict:
    np_ = lambda t: t.detach().cpu().numpy().copy()
    return {"P": {k: np_(v) for k, v in sh.P.items()}, "m": {k: np_(v) for k, v in sh.m.items()},
            "v": {k: np_(v) for k, v in sh.v.items()}}


def record(sh, out5, before) -> dict:
    """What a rank returns for one step (numpy copies)."""
    np_ = lambda t: t.detach().cpu().numpy().copy()
    return dict(out5=np_(out5), rows=np_(sh.rows), idx=np_(sh.idx), grads={k: np_(v) for k, v in sh.grads.items()},
                before=before, after=snapshot(sh), step=int(sh.step_dev.cpu()[0]))


def run_case(c: Case, rank: int, world: int, device, exchange="nccl", group=None) -> List[dict]:
    """Every optimiser step of case `c` on this rank, eager."""
    p = case_problem(c)
    cfg = config(c)
    steps = batches(c, p, world)
    sh = shard_problem(p, cfg, rank, world, device, c.schedule, exchange, nce=c.route.split("/")[1], group=group)
    pi = sh.pi
    out = []
    for u, po, ne, masks in steps:
        for dst, m in zip(sh.masks, masks):
            dst.copy_(pi.local(m, rank).to(device))
        sh.set_indices(u, po, ne)
        before = snapshot(sh)
        out5 = sh.run().clone()
        out.append(record(sh, out5, before))
    out.append(dict(schedule=sh.schedule, gathers=sh.n_gathers, reduce_scatters=sh.n_reduce_scatters))
    return out


# ---------------------------------------------------------------------------------------------------------------- judge
def classes(p: H.Problem, world: int, schedule: str) -> Dict[str, Dict[str, torch.Tensor]]:
    """hotstep_fp64.row_classes plus the block edges and the item rows' classes in the rank operands."""
    from mmssl_b200.parallel import RowPartition
    cls = H.row_classes(p)
    for table, n in ((H.P_EU, p.U), (H.P_EI, p.I)):
        part = RowPartition(n, world)
        m = torch.zeros(n, dtype=torch.bool)
        for r in range(world):
            lo, hi = part.bounds(r)
            if hi > lo:
                m[lo] = m[hi - 1] = True
        cls[table]["block edge"] = m
    if schedule == "reduce_scatter" and world > 1:
        split, _, heavy, _ = p.cuts
        pu = RowPartition(p.U, world)
        worst = np.zeros((world, p.I), np.int64)          # item row's stored entries in each rank's column-block operand
        seen = set()
        for g in p.coo:
            if id(g) in seen:
                continue
            seen.add(id(g))
            m = _scipy(g).tocoo()
            items, users = (m.row, m.col) if g[3] == (p.I, p.U) else (m.col, m.row)
            for r in range(world):
                lo, hi = pu.bounds(r)
                sel = (users >= lo) & (users < hi)
                worst[r] = np.maximum(worst[r], np.bincount(items[sel], minlength=p.I))
        cls[H.P_EI]["split (rank operand)"] = torch.from_numpy(((worst > split) & (worst <= heavy)).any(0))
        cls[H.P_EI]["heavy (rank operand)"] = torch.from_numpy((worst > heavy).any(0))
    return cls


def _bitwise(a, b) -> bool:
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def judge(c: Case, world: int, res: Dict[int, List[dict]], what: str = "", steps=None, first_step: int = 1) -> None:
    """Every step of every rank of case `c` against float64, and the exact invariants.  `steps`: the (users, pos, neg, masks)
    of each step when they are not ``batches(c)`` (a device sampler drew them); `first_step`: the optimiser step of the first."""
    from mmssl_b200.parallel import RowPartition
    from tests.test_gpu_zz_hotstep_fp64 import _adamw_refs, assert_update
    what = f"{what} world={world} {c.name}"
    p = case_problem(c)
    cfg = config(c)
    steps = batches(c, p, world) if steps is None else steps
    parts = {H.P_EU: RowPartition(c.U, world), H.P_EI: RowPartition(c.I, world)}
    tail = [res[r][-1] for r in range(world)]
    assert all(t["schedule"] == (c.schedule if world > 1 else "allgather") for t in tail), (what, tail)
    def full(r_blocks, k):
        part = parts[k]
        return torch.from_numpy(np.concatenate([r_blocks[r][:part.bounds(r)[1] - part.bounds(r)[0]] for r in range(world)]))

    for s, (u, po, ne, masks) in enumerate(steps):
        recs = [res[r][s] for r in range(world)]
        at = f"{what} step {s}"
        # ---- exact invariants
        for r, rec in enumerate(recs):
            for k, part in parts.items():
                n_real = part.bounds(r)[1] - part.bounds(r)[0]
                assert not rec["grads"][k][n_real:].any(), f"{at} rank {r}: padded rows of the {k} gradient are not 0"
                for st in ("P", "m", "v"):
                    assert _bitwise(rec["after"][st][k][n_real:], rec["before"][st][k][n_real:]), \
                        f"{at} rank {r}: padded rows of {st}[{k}] changed"
            for name, a, b in [("losses", rec["out5"], recs[0]["out5"]), ("self.rows", rec["rows"], recs[0]["rows"]),
                               ("batch", rec["idx"], recs[0]["idx"])] + \
                    [(f"gradient {k}", rec["grads"][k], recs[0]["grads"][k]) for k in REPLICATED] + \
                    [(f"{st}[{k}] after the step", rec["after"][st][k], recs[0]["after"][st][k]) for k in REPLICATED
                     for st in ("P", "m", "v")]:
                assert _bitwise(a, b), f"{at}: {name} differ between rank {r} and rank 0"
        assert np.array_equal(recs[0]["idx"], np.stack([u, po, ne])), at
        # ---- against float64 at the parameters the ranks held
        before = {k: (full([rec["before"]["P"][k] for rec in recs], k) if k in parts else torch.from_numpy(recs[0]["before"]["P"][k]))
                  for k in H.LIVE}
        q = p.with_batch(u, po, ne, masks=masks)
        hi, lo = H.both(q, cfg, params=before)
        route = c.route
        H.assert_losses(torch.from_numpy(recs[0]["out5"]), lo["losses"], hi["losses"], route, at)
        cq = classes(q, world, tail[0]["schedule"])
        grads = {}
        for k in H.LIVE:
            grads[k] = full([rec["grads"][k] for rec in recs], k) if k in parts else torch.from_numpy(recs[0]["grads"][k])
            H.assert_close(k, grads[k], lo["grads"][k], hi["grads"][k], route, cq.get(k), at)
        # ---- the AdamW update of every tensor, from the device's own gradient
        step = recs[0]["step"]
        assert step == s + first_step, (at, step)
        for k in H.LIVE:
            get = (lambda st, when: full([rec[when][st][k] for rec in recs], k)) if k in parts else \
                (lambda st, when: torch.from_numpy(recs[0][when][st][k]))
            p0, m0, v0 = get("P", "before"), get("m", "before"), get("v", "before")
            h64, l32 = _adamw_refs(p0, grads[k], m0, v0, step, cfg.lr, cfg.beta1, cfg.beta2, cfg.eps, cfg.weight_decay)
            assert_update(f"{at} {k}", p0, (get("P", "after"), get("m", "after"), get("v", "after")), h64, l32)


# ---------------------------------------------------------------------------------------------------------------- launch
def run_cases(cases, rank: int, world: int, device, exchange="nccl", group=None, cuts=None) -> List[List[dict]]:
    from mmssl_b200 import ops
    out = []
    for c in cases:
        if cuts is not None:
            ops.spmm_plan_set_cuts(*c.cuts)
        try:
            out.append(run_case(c, rank, world, device, exchange, group))
        finally:
            if cuts is not None:
                ops.spmm_plan_set_cuts(*H.DEFAULT_CUTS)
    return out


def gpu_cases(world: int) -> List[Case]:
    """The multi-GPU cases (both schedules are added by main)."""
    return [Case(U=1531, I=1237, d=64, B=257, modal="distinct", route="tc/auto", steps=3, kind="block edges"),
            Case(U=1531, I=1237, d=96, B=96, K=3, heads=1, modal="empty", route="simt/simt", steps=2, kind="repeated"),
            Case(U=523, I=391, d=128, B=96, modal="alias", route="simt/auto", steps=2, kind="one rank",
                 terms=(("feat_reg_decay", 391.0),)),
            Case(U=523, I=391, d=64, B=96, modal="distinct", route="tc/auto", steps=2, drop=0.0)]


def main() -> None:
    """One rank under torch.distributed.run on the GPUs: every case of gpu_cases on both schedules through the exchange of
    argv[1] ('nccl' or 'multicast'), judged on rank 0 (the ranks' records travel by gather_object); then eight replays of the
    captured multicast step and the replicated parameters compared bitwise across the ranks.  Prints one JSON line on rank 0."""
    import sys
    import torch.distributed as dist
    exchange = sys.argv[1] if len(sys.argv) > 1 else "nccl"
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    result = dict(world=world, exchange=exchange, cases=0, replays=0)
    try:
        cases = [replace(c, schedule=s) for c in gpu_cases(world) for s in ("reduce_scatter", "allgather")]
        mine = run_cases(cases, rank, world, "cuda", exchange)
        every = [None] * world if rank == 0 else None
        dist.gather_object(mine, every, dst=0)
        if rank == 0:
            for j, c in enumerate(cases):
                judge(c, world, {r: every[r][j] for r in range(world)}, what=exchange)
            result["cases"] = len(cases)
        if exchange == "multicast":
            recs = replay_records(Case(U=1531, I=1237, d=64, B=257, modal="distinct", route="tc/auto"), rank, world, "cuda", n=8)
            every = [None] * world if rank == 0 else None
            dist.gather_object(recs, every, dst=0)
            if rank == 0 and recs is None:
                result["replays"] = None
            elif rank == 0:
                for s in range(len(recs)):
                    for r in range(1, world):
                        for k in REPLICATED:
                            for st in ("P", "m", "v"):
                                assert _bitwise(every[r][s][st][k], every[0][s][st][k]), f"replay {s}: {st}[{k}] differ, rank {r}"
                        assert _bitwise(every[r][s]["out5"], every[0][s]["out5"]), f"replay {s}: losses differ, rank {r}"
                result["replays"] = len(recs)
        if rank == 0:
            result["ledger"] = [[*k, *v] for k, v in sorted(H.LEDGER.items())]
            print(json.dumps(result), flush=True)
    finally:
        dist.barrier()
        dist.destroy_process_group()


def replay_records(c: Case, rank: int, world: int, device, n: int = 8) -> List[dict]:
    """`n` replays of the captured multicast step (batch set between replays): replicated P / m / v and losses after each;
    None where the system has no multicast address."""
    p = case_problem(c)
    steps = batches(replace(c, steps=n), p, world)
    sh = shard_problem(p, config(c), rank, world, device, c.schedule, "multicast", nce=c.route.split("/")[1])
    if sh.ar_rows is None:                  # no NVSwitch multicast address: the step cannot be captured
        return None
    sh.capture(warmup=1)
    out = []
    for u, po, ne, masks in steps:
        for dst, m in zip(sh.masks, masks):
            dst.copy_(sh.pi.local(m, rank).to(device))
        sh.set_indices(u, po, ne)
        out5 = sh.replay().clone()
        snap = snapshot(sh)
        out.append({"out5": out5.cpu().numpy().copy(), **{st: {k: snap[st][k] for k in REPLICATED} for st in ("P", "m", "v")}})
    return out


if __name__ == "__main__":
    main()
