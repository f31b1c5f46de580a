#!/usr/bin/env python
"""Key numbers of an ncu report (`ncu --set full ... -o report`), read here without a GPU:
    python tools/ncu_summary.py report.ncu-rep [report2.ncu-rep ...]
duration, launch shape, registers, shared memory, executed warp instructions, issue-slot utilisation, stall reasons per issued
instruction, pipe utilisation, DRAM bytes (traffic)."""
import csv
import subprocess
import sys

KEYS = [
    ("duration_us", "gpu__time_duration.sum"),
    ("grid", "launch__grid_size"), ("block", "launch__block_size"), ("registers", "launch__registers_per_thread"),
    ("smem_dynamic_KB", "launch__shared_mem_per_block_dynamic"), ("occupancy_limit_regs", "launch__occupancy_limit_registers"),
    ("occupancy_limit_smem", "launch__occupancy_limit_shared_mem"),
    ("warp_instructions", "smsp__inst_executed.sum"),
    ("issue_active_pct", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
    ("warps_per_scheduler", "smsp__warps_active.avg.per_cycle_active"), ("eligible_per_scheduler", "smsp__warps_eligible.avg.per_cycle_active"),
    ("active_threads_per_inst", "smsp__thread_inst_executed_per_inst_executed.ratio"),
    ("achieved_occupancy_pct", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("dram_read_bytes", "dram__bytes_read.sum"), ("dram_write_bytes", "dram__bytes_write.sum"),
    ("dram_throughput_pct", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
    ("pipe_fma_pct", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"), ("pipe_alu_pct", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"),
    ("pipe_lsu_pct", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active"),
]


def load(rep):
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    hdr, units = rows[0], rows[1]
    out = []
    for r in rows[2:]:
        if len(r) == len(hdr):
            out.append((dict(zip(hdr, r)), dict(zip(hdr, units))))
    return out


for rep in sys.argv[1:]:
    for d, u in load(rep):
        print(f"## {rep}: {d.get('Kernel Name', '?')[:110]}")
        for name, key in KEYS:
            if key in d:
                print(f"  {name:26s} {d[key]} {u.get(key, '')}")
        stalls = {k.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""): float(v) for k, v in d.items()
                  if "average_warps_issue_stalled" in k and k.endswith("_per_issue_active.ratio") and v not in ("", "n/a")}
        top = sorted(stalls.items(), key=lambda kv: -kv[1])[:7]
        print("  stalls per issued instr   " + ", ".join(f"{k} {v:.2f}" for k, v in top))
