#!/usr/bin/env python3
"""Summarise .ncu-rep captures into a small text file.
usage: ncu_summary.py out.md report1.ncu-rep [report2 ...]"""
import csv, io, subprocess, sys
KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "sm__warps_active.avg.per_cycle_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.per_cycle_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__sass_average_branch_targets_threads_uniform.pct",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "l1tex__throughput.avg.pct_of_peak_sustained_active", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__inst_executed.sum"]
out = open(sys.argv[1], "w")
for rep in sys.argv[2:]:
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        out.write(f"## {rep.split('/')[-1]} :: {r[hdr.index('Kernel Name')]}\n")
        for k in KEYS:
            if k in hdr:
                out.write(f"  {k:72s} {r[hdr.index(k)]} {units[hdr.index(k)]}\n")
        st = [(float(r[i]), k) for i, k in enumerate(hdr) if k.startswith("smsp__pcsamp_warps_issue_stalled_")
              and not k.endswith("_not_issued") and r[i] not in ("", "n/a")]
        tot = sum(s for s, _ in st) or 1
        out.write("  stall samples: " + ", ".join(f"{k[33:]} {100 * s / tot:.0f}%" for s, k in sorted(st, reverse=True)[:7]) + "\n\n")
out.close()
print(open(sys.argv[1]).read())
