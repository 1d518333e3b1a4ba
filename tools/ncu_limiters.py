#!/usr/bin/env python
"""What bounds each kernel, from `ncu --set full` captures: issue-slot use, the top warp-stall reasons (warps stalled per issued
instruction), achieved occupancy, cache hit rates and the DRAM / tensor-pipe / FMA-pipe utilisation, one row per kernel.

    python tools/ncu_limiters.py a.ncu-rep [b.ncu-rep ...] > kernel_limiters.md
"""
import csv
import os
import re
import subprocess
import sys
from collections import OrderedDict

STALL = "smsp__average_warps_issue_stalled_{}_per_issue_active.ratio"
REASONS = ["long_scoreboard", "short_scoreboard", "wait", "barrier", "membar", "mio_throttle", "lg_throttle", "math_pipe_throttle",
           "tex_throttle", "not_selected", "dispatch_stall", "no_instruction", "branch_resolving", "sleeping", "drain", "misc"]
COLS = OrderedDict([
    ("us", "gpu__time_duration.sum"), ("regs", "launch__registers_per_thread"),
    ("warps active %", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("issue %", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
    ("DRAM %", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
    ("L2 hit %", "lts__t_sector_hit_rate.pct"), ("L1 hit %", "l1tex__t_sector_hit_rate.pct"),
    ("tensor %", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
    ("FMA %", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active"),
])


def short(name):
    name = re.sub(r"^void\s+", "", name)
    name = re.sub(r"\(.*$", "", name)
    return re.sub(r"^ctr::", "", name)


def rows_of(rep):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr = rows[0]
    for r in rows[2:]:
        yield dict(zip(hdr, r))


def num(x):
    try:
        return float(str(x).replace(",", ""))
    except ValueError:
        return float("nan")


def main(reps):
    print("| capture | kernel | " + " | ".join(COLS) + " | top stalls (warps stalled per issued instruction) |")
    print("|---|---|" + "---|" * (len(COLS) + 1))
    for rep in reps:
        seen = {}
        for r in rows_of(rep):
            k = short(r["Kernel Name"])
            seen.setdefault(k, []).append(r)
        for k, rs in seen.items():
            r = min(rs, key=lambda x: num(x["gpu__time_duration.sum"]))      # the fastest (warm) launch of this kernel
            stalls = sorted(((num(r.get(STALL.format(s), "nan")), s) for s in REASONS if STALL.format(s) in r), reverse=True)
            top = ", ".join(f"{s} {v:.2f}" for v, s in stalls[:3] if v == v and v > 0.005)
            cells = []
            for label, m in COLS.items():
                v = num(r.get(m, "nan"))
                cells.append("–" if v != v else (f"{v:.0f}" if label == "regs" else f"{v:.1f}"))
            print(f"| `{os.path.basename(rep)}` | `{k}` ×{len(rs)} | " + " | ".join(cells) + f" | {top} |")


if __name__ == "__main__":
    main(sys.argv[1:])
