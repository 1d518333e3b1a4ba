#!/usr/bin/env python
"""Summarise an Nsight Compute report (.ncu-rep) into a small CSV.

    python tools/ncu_summary.py prof.ncu-rep prof.summary.csv
"""
import csv
import subprocess
import sys

METRICS = [
    "Kernel Name", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__cycles_active.avg",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor.sum", "smsp__inst_executed.sum",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "smsp__cycles_active.avg", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    cols = [(m, hdr.index(m)) for m in METRICS if m in hdr]
    with open(out, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow([f"{m} [{units[i]}]" if units[i] else m for m, i in cols])
        for r in rows[2:]:
            w.writerow([r[i] for _, i in cols])
    print(open(out).read())


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
