"""Summarise an `ncu --page raw --csv` export: one block of headline metrics per captured kernel.

    python tools/ncu_csv_summary.py <ncu --csv export> [kernel-name-substring]"""
import csv
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__compute_memory_throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "l1tex__t_bytes.sum", "l1tex__throughput.avg.pct_of_peak_sustained_active", "l1tex__t_sector_hit_rate.pct",
    "sm__inst_executed.sum", "sm__inst_executed_pipe_tensor.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.sum", "smsp__issue_active.avg.pct", "smsp__inst_executed.avg.per_cycle_active",
    "sm__cycles_active.avg", "sm__cycles_elapsed.max", "smsp__cycles_active.avg",
]
STALL = "smsp__average_warps_issue_stalled_"        # ..._per_issue_active.ratio  (warp-state sampling section)


def main():
    rows = list(csv.reader(open(sys.argv[1])))
    want = sys.argv[2] if len(sys.argv) > 2 else ""
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    for r in rows[2:]:
        name = r[idx["Kernel Name"]]
        if want not in name:
            continue
        print(f"== {name[:110]}  grid {r[idx['Grid Size']]} block {r[idx['Block Size']]}")
        for k in KEYS:
            if k in idx and r[idx[k]] != "":
                print(f"   {k:72s} {r[idx[k]]:>16s} {units[idx[k]]}")
        stalls = []
        for h, i in idx.items():
            if h.startswith(STALL) and h.endswith("_per_issue_active.ratio") and r[i] not in ("", "0"):
                try:
                    stalls.append((float(r[i].replace(",", "")), h[len(STALL):-len("_per_issue_active.ratio")]))
                except ValueError:
                    pass
        stalls.sort(reverse=True)
        if stalls:
            print("   warp stall reasons (avg warps stalled per issue): " + ", ".join(f"{n} {v:.2f}" for v, n in stalls[:7]))


if __name__ == "__main__":
    main()
