"""Row-sharded device sampler (sampler.ShardedTripleSampler) on the GPUs of one box.  One JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/rowshard_sampler_bench.py check
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/rowshard_sampler_bench.py [--iters K]
    (or plain `python tools/rowshard_sampler_bench.py ...` for one GPU)

check   every rank's [3, B] batch against DeviceTripleSampler on the whole training matrix (built on rank 0), both sampler paths,
        a permutation and with replacement, several steps, at Baby and 1M users; exit code 1 unless all are bitwise equal.
timing  sample_into per call (CUDA events around K calls, max over ranks) at B = 1024 / 4096 / 16384 for 19 445 (Baby),
        1M and 10M users, and the captured row-sharded step at Sports with the in-graph draw against the same captured step
        fed one batch (world 1, or the multicast exchange on several GPUs).
The user rows are a pattern computed on the device from the global user id (device_rows): a rank builds its own block, no rank
ever holds the 10M-row matrix, and the rows do not depend on the world size."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

MAX_DEG = 16
SIZES = {"baby": (19445, 7050), "syn1m": (1_000_000, 200_000), "syn10m": (10_000_000, 1_000_000)}


def _mix(x: torch.Tensor, seed: int) -> torch.Tensor:
    """A non-negative 31-bit hash of int64 x (wrapping int64 arithmetic, identical on every device)."""
    x = x * 6364136223846793005 + (seed * 1442695040888963407 & 0x7FFFFFFFFFFFFFFF)
    x = x ^ (x >> 29)
    x = x * 3935559000370003845
    return (x >> 33) & 0x7FFFFFFF


def device_rows(n_users: int, n_items: int, lo: int, hi: int, seed: int, device, block: int = None):
    """dataset.CsrBlock of the users [lo, hi) of a pattern: user u has mix(u) % 17 items (about 6% have none), item k of the
    row in the k-th of 16 equal item ranges, so rows are sorted and distinct.  Device tensors."""
    from mmssl_b200.dataset import CsrBlock
    u = torch.arange(lo, hi, dtype=torch.int64, device=device)
    deg = _mix(u, seed) % (MAX_DEG + 1)
    indptr = torch.zeros(hi - lo + 1, dtype=torch.int64, device=device)
    indptr[1:] = torch.cumsum(deg, 0)
    row = torch.repeat_interleave(torch.arange(hi - lo, device=device), deg)
    k = torch.arange(row.numel(), dtype=torch.int64, device=device) - indptr[row]
    stride = n_items // MAX_DEG
    items = k * stride + _mix(u[row] * (MAX_DEG + 1) + k, seed + 1) % stride
    return CsrBlock(indptr, items.to(torch.int32), None, (block or hi - lo, n_items), lo, hi)


def to_scipy(blk) -> sp.csr_matrix:
    ip, ix = blk.indptr.cpu().numpy(), blk.indices.cpu().numpy()
    return sp.csr_matrix((np.ones(ix.size, np.float32), ix, ip), shape=(len(ip) - 1, blk.shape[1]))


def _env():
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    return rank, world, dev


def _card():
    try:
        q = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def _exchanges(world):
    """The exchanges a multi-GPU box offers: NCCL always, the multicast kernel when symmetric memory has a multicast address."""
    return ["nccl", "multicast"] if world > 1 else ["nccl"]


def check(rank, world, dev):
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.sampler import DeviceTripleSampler, ShardedTripleSampler
    bad, n_cmp = [], 0
    for name in ("baby", "syn1m"):
        U, I = SIZES[name]
        pu = RowPartition(U, world)
        lo, hi = pu.bounds(rank)
        full = DeviceTripleSampler(to_scipy(device_rows(U, I, 0, U, 5, dev)), device=dev, seed=11) if rank == 0 else None
        n_exist = full.exist.numel() if rank == 0 else None
        for ex in _exchanges(world):
            smp = ShardedTripleSampler(device_rows(U, I, lo, hi, 5, dev, pu.block), pu, rank, device=dev, seed=11, exchange=ex)
            for b in (1, 1000, 1024, 1025, 4096, 16384, smp.n_exist, smp.n_exist + 1):
                for step in (0, 1, 9):
                    got = smp.sample_into(torch.full((3, b), -1, dtype=torch.int64, device=dev), step=step)
                    ex_used = ("multicast" if smp.ar.get(b) is not None else "nccl") if world > 1 else "none"
                    if rank == 0:
                        want = full.sample_into(torch.zeros(3, b, dtype=torch.int64, device=dev), step=step)
                        n_cmp += 1
                        if not torch.equal(got, want):
                            bad.append(f"{name}/{ex_used}: B={b} step={step}")
            if rank == 0 and smp.n_exist != n_exist:
                bad.append(f"{name}: n_exist {smp.n_exist} vs {n_exist}")
    torch.cuda.synchronize()
    return {"mode": "check", "n_gpus": world, "exchanges": _exchanges(world), "comparisons": n_cmp, "mismatches": bad,
            "check": not bad}


def _time(fn, iters, dev):
    for _ in range(5):
        fn()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / iters


def _max_over_ranks(v, world, dev):
    t = torch.tensor([v], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def timing(rank, world, dev, iters):
    from mmssl_b200.parallel import RowPartition
    from mmssl_b200.sampler import ShardedTripleSampler
    res = {"mode": "timing", "n_gpus": world, "card": _card(), "exchange": "multicast" if world > 1 else "none", "sample_into_ms": {}}
    for name, (U, I) in SIZES.items():
        pu = RowPartition(U, world)
        lo, hi = pu.bounds(rank)
        smp = ShardedTripleSampler(device_rows(U, I, lo, hi, 5, dev, pu.block), pu, rank, device=dev, seed=11,
                                   exchange="multicast" if world > 1 else "nccl")
        row = {"n_exist": smp.n_exist}
        for b in (1024, 4096, 16384):
            out = torch.zeros(3, b, dtype=torch.int64, device=dev)
            step = torch.zeros(1, dtype=torch.int32, device=dev)
            smp.reserve(b)

            def call():
                smp.sample_into(out, step_dev=step)
                step.add_(1)
            row[f"B{b}"] = round(_max_over_ranks(_time(call, iters, dev), world, dev), 4)
        res["sample_into_ms"][name] = row
        del smp
        torch.cuda.empty_cache()
    res["sports_step"] = step_ab(rank, world, dev, iters)
    return res


def step_ab(rank, world, dev, iters, batch=4096):
    """The captured row-sharded step at Sports, B = 4096: with the in-graph draw against the same step fed one fixed batch.
    Alternated twice (A B A B) so that drift of the shared machine shows as a spread."""
    import bench
    from mmssl_b200.dataset import CsrBlock
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.parallel import shard_rows_scipy
    from mmssl_b200.rowshard_step import RowShardedHotStep, shard_problem
    from mmssl_b200.sampler import ShardedTripleSampler
    ds, P_cpu, feats_cpu, _, _ = bench.build_problem("sports", 2022, None)
    cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=batch)
    steps = {}
    for mode in ("sampler", "fixed"):
        Pl, fl, gl, pu, pi = shard_problem(P_cpu, feats_cpu, ds.ui_norm, ds.iu_norm, rank, world, dev)
        smp = None
        if mode == "sampler":
            lo, hi = pu.bounds(rank)
            blk = shard_rows_scipy(ds.train, pu, rank)
            smp = ShardedTripleSampler(CsrBlock(blk.indptr.astype(np.int64), blk.indices.astype(np.int32), None, blk.shape, lo, hi), pu,
                                       rank, device=dev, seed=2022, exchange="multicast" if world > 1 else "nccl")
        sh = RowShardedHotStep(Pl, fl, gl, cfg, batch, pu, pi, rank, exchange="multicast" if world > 1 else "nccl", sampler=smp)
        if smp is not None:
            smp.sample_into(sh.idx, step=0)
            fixed = sh.idx.clone()
        else:
            sh.idx.copy_(fixed)
        sh.optimizer_step = False          # the same parameters every replay: a steady state to time
        sh.capture()
        steps[mode] = sh
    ms = {"sampler": [], "fixed": []}
    for _ in range(2):
        for mode in ("sampler", "fixed"):
            ms[mode].append(round(_max_over_ranks(_time(steps[mode].replay, iters, dev), world, dev), 4))
    return {"config": "sports", "batch": batch, "ms_per_step_in_graph_draw": ms["sampler"], "ms_per_step_fixed_batch": ms["fixed"],
            "draw_cost_ms": round(min(ms["sampler"]) - min(ms["fixed"]), 4)}


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    iters = int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 200
    rank, world, dev = _env()
    res = check(rank, world, dev) if "check" in args else timing(rank, world, dev, iters)
    if rank == 0:
        print(json.dumps(res))
    ok = res.get("check", True)
    if world > 1:
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
