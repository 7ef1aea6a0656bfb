"""Thread-count sweep of the CPU baseline (bench.py's cpu_baseline leg): torch's sparse kernels get slower with more threads on
the GPU hosts, so the baseline is reported at its best setting."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import bench
name = sys.argv[1] if len(sys.argv) > 1 else "baby"
for nt in (8, 16, 32, 64, 128):
    r = bench.cpu_baseline(name, 2022, 3, bench.BATCH, threads=nt)
    print(json.dumps({"threads": r["cores"], "s_per_step": r["s_per_step"], "sample": r["sample"]}), flush=True)
