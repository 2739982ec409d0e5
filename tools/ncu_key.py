#!/usr/bin/env python3
"""Key numbers of an .ncu-rep (read here, no GPU): python tools/ncu_key.py x.ncu-rep"""
import csv
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__cycles_active.avg", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed_pipe_alu.sum", "smsp__inst_executed_pipe_fma.sum",
        "smsp__inst_executed_pipe_fmaheavy.sum", "smsp__inst_executed_pipe_fmalite.sum", "smsp__inst_executed_pipe_xu.sum",
        "smsp__inst_executed_pipe_lsu.sum", "smsp__inst_executed_pipe_uniform.sum", "smsp__inst_executed_pipe_cbu.sum",
        "smsp__inst_executed_pipe_adu.sum"]
rows = list(csv.reader(subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout.splitlines()))
hdr, units = rows[0], rows[1]
for r in rows[2:]:
    print("==", r[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "")
    for i, h in enumerate(hdr):
        if h in WANT or ("issue_stalled" in h and h.endswith("per_issue_active.ratio")):
            try:
                v = float(r[i])
            except ValueError:
                continue
            if "issue_stalled" in h and v < 0.05:
                continue
            print(f"  {h:90s} {units[i]:12s} {r[i]}")
