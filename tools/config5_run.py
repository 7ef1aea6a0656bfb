"""BASELINE config 5 (synthetic bipartite 10M x 1M, 200M edges, d = 256, V4096/T1024) -- or any --users/--items/--edges -- as the
row-sharded whole hot step on the GPUs of one box (VERDICT r1 #10).  Everything is generated ON THE DEVICE, per rank: the host
generator of mmssl_b200/synthetic.py would take minutes per rank at this size.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/config5_run.py [--users N --items N --edges N --embed-size D]

Every rank draws the same edge list (same seed): user degrees ~ lognormal(sigma = 1), item endpoints ~ Zipf(1.0) over a random
permutation, duplicate (u, i) pairs dropped (so the edge count ends slightly below the request); values = the reference's
csr_norm(mean_flag=True) (main.py:89-103): (deg_row + 1e-8)^-1/2 on each side.  It keeps its row blocks (and the column blocks of
the partial-product schedule), its rows of the features / tables, and runs RowShardedHotStep (multicast exchange, reduce-scatter
schedule, CUDA graph).  Prints one JSON line (rank 0): ms/step, exchanges and bytes per step, peak memory per rank.
No 1-GPU twin is built at this size: parity of the same code path is checked at Sports / 1M x 200k by bench.py --gpus N.
By default every step trains on one batch drawn once from the edge list.  With --sampler device each rank builds the training rows
of its user block from the edges it keeps, and every step (every graph replay) draws a fresh batch of Data.sample on the device
(sampler.ShardedTripleSampler: bitwise the one-GPU device sampler's batch at that step, at any world size)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--users", type=int, default=10_000_000)
ap.add_argument("--items", type=int, default=1_000_000)
ap.add_argument("--edges", type=int, default=200_000_000)
ap.add_argument("--embed-size", dest="d", type=int, default=256)
ap.add_argument("--dv", type=int, default=4096)
ap.add_argument("--dt", type=int, default=1024)
ap.add_argument("--layers", type=int, default=2)
ap.add_argument("--batch", type=int, default=1024)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--seed", type=int, default=2022)
ap.add_argument("--no-graph", action="store_true")
ap.add_argument("--sampler", choices=("fixed", "device"), default="fixed",
                help="fixed: one batch for every step; device: a fresh batch per step, drawn on the rank that holds the user's row")
a = ap.parse_args()

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)

from mmssl_b200.engine import LIVE, P_EI, P_EU, FeatureStore  # noqa: E402
from mmssl_b200.graph import SparseOperand  # noqa: E402
from mmssl_b200.hotstep import HotStepConfig  # noqa: E402
from mmssl_b200.parallel import RowPartition  # noqa: E402
from mmssl_b200.rowshard_step import RowBlockGraph, RowShardedHotStep  # noqa: E402

t0 = time.perf_counter()
U, I, d = a.users, a.items, a.d
g = torch.Generator(device=dev).manual_seed(a.seed)
# ---- the edge list (identical on every rank)
w = torch.exp(torch.randn(U, generator=g, device=dev))
deg = torch.clamp((w / w.sum() * a.edges).floor().long(), min=1, max=max(1, I // 4))
users = torch.repeat_interleave(torch.arange(U, device=dev), deg)
del w, deg
pw = 1.0 / torch.arange(1, I + 1, device=dev, dtype=torch.float64)
cdf = torch.cumsum(pw / pw.sum(), 0).float()
perm = torch.randperm(I, generator=g, device=dev)
items = torch.empty_like(users)
CH = 50_000_000
for s in range(0, users.numel(), CH):                   # in chunks: bounded temporaries
    r = torch.rand(min(CH, users.numel() - s), generator=g, device=dev)
    items[s:s + CH] = perm[torch.searchsorted(cdf, r).clamp_(max=I - 1)]
del cdf, perm, pw
keys = torch.unique(users * I + items)                  # sorted by (user, item), duplicates dropped
del users, items
rows, cols = keys // I, keys % I
del keys
nnz = int(rows.numel())
deg_u = torch.bincount(rows, minlength=U).float()
deg_i = torch.bincount(cols, minlength=I).float()
v_ui = (deg_u[rows] + 1e-8).pow(-0.5)                   # A_ui = D_u^-1/2 R
v_iu = (deg_i[cols] + 1e-8).pow(-0.5)                   # A_iu = D_i^-1/2 R^T
del deg_u, deg_i
pu, pi = RowPartition(U, world), RowPartition(I, world)
ulo, uhi = pu.bounds(rank)
ilo, ihi = pi.bounds(rank)


def operand(r, c, v, n_rows, n_cols):
    o = SparseOperand(r.contiguous(), c.contiguous(), v.contiguous(), n_rows, n_cols)
    o.tighten()
    return o


mu = (rows >= ulo) & (rows < uhi)                       # edges whose user this rank owns
mi = (cols >= ilo) & (cols < ihi)                       # edges whose item this rank owns
hu, hi_ = pu.world * pu.block, pi.world * pi.block
# A_ui [U x I]: rows u, cols i
g_ui = RowBlockGraph(operand(rows[mu] - ulo, cols[mu], v_ui[mu], pu.block, I),                     # A_ui[U_r, :]
                     operand(cols[mi] - ilo, rows[mi], v_ui[mi], pi.block, U),                     # (A_ui^T)[I_r, :]
                     (pu.block, pi.block), nnz,
                     fwd_part=operand(rows[mi], cols[mi] - ilo, v_ui[mi], hu, pi.block),           # A_ui[:, I_r]   (unused by the schedule)
                     bwd_part=operand(cols[mu], rows[mu] - ulo, v_ui[mu], hi_, pu.block))          # (A_ui^T)[:, U_r]
# A_iu [I x U]: rows i, cols u
g_iu = RowBlockGraph(operand(cols[mi] - ilo, rows[mi], v_iu[mi], pi.block, U),                     # A_iu[I_r, :]
                     operand(rows[mu] - ulo, cols[mu], v_iu[mu], pu.block, I),                     # (A_iu^T)[U_r, :]
                     (pi.block, pu.block), nnz,
                     fwd_part=operand(cols[mu], rows[mu] - ulo, v_iu[mu], hi_, pu.block),          # A_iu[:, U_r]
                     bwd_part=operand(rows[mi], cols[mi] - ilo, v_iu[mi], hu, pi.block))           # (A_iu^T)[:, I_r] (unused)
# a batch of (user, pos, neg) triples (global ids, identical on every rank)
bu = torch.randperm(U, generator=g, device=dev)[:a.batch]
first = torch.searchsorted(rows, bu)
pos = cols[first.clamp_(max=nnz - 1)]
neg = torch.randint(0, I, (a.batch,), generator=g, device=dev)
smp = None
if a.sampler == "device":                               # the rank's training rows: its edges, sorted by (user, item) already
    from mmssl_b200.dataset import CsrBlock  # noqa: E402
    from mmssl_b200.sampler import ShardedTripleSampler  # noqa: E402
    indptr = torch.zeros(pu.block + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(torch.bincount(rows[mu] - ulo, minlength=pu.block), 0)
    blk = CsrBlock(indptr.cpu().numpy(), cols[mu].to(torch.int32).cpu().numpy(), None, (pu.block, I), ulo, uhi)
    smp = ShardedTripleSampler(blk, pu, rank, device=dev, seed=a.seed, exchange="multicast" if world > 1 else "nccl")
    del indptr, blk
del rows, cols, v_ui, v_iu, mu, mi
torch.cuda.empty_cache()

# ---- parameters and features of this rank
gr = torch.Generator(device=dev).manual_seed(a.seed + 1000 * rank + 1)
xav = lambda r, c, fan_r=None: (torch.rand(r, c, generator=gr, device=dev) * 2 - 1) * (6.0 / ((fan_r or r) + c)) ** 0.5
gs = torch.Generator(device=dev).manual_seed(a.seed + 7)         # replicated small parameters: same values on every rank
xs = lambda r, c: (torch.rand(r, c, generator=gs, device=dev) * 2 - 1) * (6.0 / (r + c)) ** 0.5
P = {"image_trans.weight": xs(d, a.dv), "image_trans.bias": torch.zeros(d, device=dev), "text_trans.weight": xs(d, a.dt),
     "text_trans.bias": torch.zeros(d, device=dev), "weight_dict.w_self_attention_cat": xs(4 * d, d),
     P_EU: xav(pu.block, d, U), P_EI: xav(pi.block, d, I)}
feats = []
for D in (a.dv, a.dt):
    f = torch.randn(pi.block, D, generator=gr, device=dev)
    f[ihi - ilo:] = 0
    feats.append(FeatureStore(f, keep_fp32=False))
    del f
gen_s = time.perf_counter() - t0

cfg = HotStepConfig(embed_size=d, n_layers=a.layers, batch_size=a.batch)
sh = RowShardedHotStep(P, feats, (g_ui, g_iu, g_ui, g_iu, g_ui, g_iu), cfg, a.batch, pu, pi, rank,
                       exchange="multicast" if world > 1 else "nccl", schedule="reduce_scatter", sampler=smp)
sh.set_indices(bu, pos, neg)                             # (overwritten by every step when the sampler draws the batch)
out = sh.run().clone()                                   # first eager step (creates the symmetric tables)
torch.cuda.synchronize()
captured = False
if not a.no_graph and world > 1:
    sh.capture()
    captured = True
step = sh.replay if captured else sh.run
for _ in range(2):
    step()
torch.cuda.synchronize()
if world > 1:
    dist.barrier()
sh.n_gathers = sh.gathered_bytes = sh.n_reduce_scatters = 0
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(a.steps):
    step()
e1.record()
torch.cuda.synchronize()
ms = torch.tensor([e0.elapsed_time(e1) / a.steps], device=dev)
peak = torch.tensor([torch.cuda.max_memory_allocated(dev) / 2 ** 30], device=dev)
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    dist.all_reduce(peak, op=dist.ReduceOp.MAX)
if not captured:
    gath, rsc, gbytes = sh.n_gathers // a.steps, sh.n_reduce_scatters // a.steps, sh.gathered_bytes / a.steps
else:
    sh.n_gathers = sh.gathered_bytes = sh.n_reduce_scatters = 0
    sh.run(); torch.cuda.synchronize()
    gath, rsc, gbytes = sh.n_gathers, sh.n_reduce_scatters, float(sh.gathered_bytes)
if rank == 0:
    print(json.dumps({"workload": f"synthetic bipartite {U}x{I}, {nnz} edges (requested {a.edges}), d={d}, {a.layers}-layer GCN, V{a.dv}/T{a.dt}, global B={a.batch}",
                      "batches": "device sampler, fresh per step" if smp is not None else "one fixed batch",
                      "n_gpus": world, "scheme": "row-sharded whole hot step (multicast exchange, reduce-scatter schedule)", "cuda_graph": captured,
                      "ms_per_step": round(float(ms), 3), "triples_per_s": round(a.batch / float(ms) * 1e3, 1), "loss_first_step": [round(float(x), 6) for x in out],
                      "all_gathers_per_step": int(gath), "reduce_scatters_per_step": int(rsc), "bytes_received_per_rank_per_step": int(gbytes),
                      "peak_GiB_per_rank": round(float(peak), 2), "generation_s": round(gen_s, 1)}))
if world > 1:
    dist.destroy_process_group()
