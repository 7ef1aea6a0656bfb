"""Writes tests/golden/device_sampler_batches.npz: batches of the device triple sampler (mmssl_b200/csrc/sampler.cu) as the
kernels drew them before the claim finish and the complement fallback existed, executed by the cuemu emulator.  The sampler
is integer-only, so these are the H100's bits too.  Every recorded batch completes its claim rounds and finds each negative
within the rejection cap, so the fixed kernels must still draw it bit for bit (tests/test_cpu_sampler_model.py checks the
model against it, the emulator and GPU tests check the kernels against the model).

    python -m tests.golden.make_golden_device_sampler"""
import json
import os

import numpy as np
import scipy.sparse as sp

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "device_sampler_batches.npz")
SEEDS = [0, 2022, 2 ** 63 + 5, 2 ** 64 - 1]
STEPS = [0, 1, 2 ** 31 - 1]


def matrices():
    """name -> csr.  'small': 300 users (every 7th empty), 40 items, rows of 1..8 items; 'dense': 90 users of 25 items with
    rows of 1..24 items (many rejections, never 4096 in a row)."""
    rng = np.random.default_rng(11)
    rows, cols = [], []
    for u in range(300):
        if u % 7 == 3:
            continue
        it = rng.choice(40, size=int(rng.integers(1, 9)), replace=False)
        rows += [u] * len(it)
        cols += it.tolist()
    small = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(300, 40))
    rows, cols = [], []
    for u in range(90):
        it = rng.choice(25, size=int(rng.integers(1, 25)), replace=False)
        rows += [u] * len(it)
        cols += it.tolist()
    dense = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(90, 25))
    for m in (small, dense):
        m.sort_indices()
    return {"small": small, "dense": dense}


def cases(n_exist):
    """(path, batch) per matrix: the one-CTA kernel well below n_exist and with replacement, the select at every size class."""
    one = [("one", b) for b in (1, 2, 33, n_exist // 4, n_exist + 1)]
    sel = [("multi", b) for b in (1, 7, n_exist // 2, n_exist - 1, n_exist, n_exist + 1)]
    return one + sel


def main():
    import torch
    from mmssl_b200 import _lib
    from mmssl_b200._lib import ptr
    from mmssl_b200.sampler import DeviceTripleSampler
    from tests.cuemu import harness

    class MP:
        def setattr(self, o, n, v):
            setattr(o, n, v)
    harness.set_order("fwd")
    lib = harness.emulated_device(MP())
    arrays, meta = {}, []
    for name, m in matrices().items():
        arrays[f"{name}_indptr"] = m.indptr.astype(np.int64)
        arrays[f"{name}_indices"] = m.indices.astype(np.int64)
        arrays[f"{name}_shape"] = np.array(m.shape, np.int64)
        for seed in SEEDS:
            smp = DeviceTripleSampler(m, device="cpu", seed=seed)
            n_exist = smp.exist.numel()
            for path, b in cases(n_exist):
                for step in STEPS:
                    out = torch.zeros(3, b, dtype=torch.int64)
                    if path == "one":
                        smp.sample_into(out, step=step)
                    else:
                        nbytes = lib.mmssl_sampler_workspace_bytes(n_exist, b)
                        ws = torch.zeros(max(nbytes, 1), dtype=torch.uint8)
                        _lib.check(lib.mmssl_sample_triples_multi(ptr(smp.indptr), ptr(smp.indices), ptr(smp.exist), n_exist, smp.n_items,
                                                                  b, seed, None, step, ptr(ws), ws.numel(), ptr(out[0]), ptr(out[1]),
                                                                  ptr(out[2]), None))
                    key = f"b{len(meta)}"
                    arrays[key] = out.numpy().copy()
                    meta.append({"key": key, "matrix": name, "path": path, "batch": b, "seed": str(seed), "step": step})
    arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **arrays)
    print(f"{OUT}: {len(meta)} batches")


if __name__ == "__main__":
    main()
