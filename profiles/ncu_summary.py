#!/usr/bin/env python3
"""Summarise an .ncu-rep (raw page) into a handful of numbers: time, DRAM traffic, issue and pipe utilisation, stalls.
Usage: python profiles/ncu_summary.py report.ncu-rep [kernel-regex]"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, data = rows[0], rows[1], rows[2:]
want = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.per_cycle_active",
    "smsp__inst_executed.sum", "sm__inst_executed.avg.per_cycle_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
    "memory_l1_wavefronts_shared", "memory_l1_wavefronts_shared_ideal",
    "l1tex__t_sectors_pipe_lsu_mem_local_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_local_op_st.sum",
    "l1tex__m_xbar2l1tex_read_bytes_mem_global_op_tma_ld.sum",
]
want += [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled") and h.endswith("per_issue_active.ratio")]
name_i = hdr.index("Kernel Name")
for r in data:
    print("kernel:", r[name_i][:80])
    for w in want:
        if w in hdr:
            i = hdr.index(w)
            print(f"  {w:85s} {r[i]:>16s} {units[i]}")
