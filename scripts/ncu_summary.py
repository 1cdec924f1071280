#!/usr/bin/env python
"""scripts/ncu_summary.py -- selected metrics of every kernel in an .ncu-rep (ncu --set full) as JSON, plus the DRAM bytes per
launch.  Usage: python scripts/ncu_summary.py REP.ncu-rep > top_kernels.json"""
import csv
import json
import subprocess
import sys

WANT = ["Kernel Name", "gpu__time_duration.sum", "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__cluster_dim_x",
        "launch__shared_mem_per_block_dynamic", "dram__bytes_read.sum", "dram__bytes_write.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.sum", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor_subpipe_dmma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio"]

out = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout.splitlines()
rows = list(csv.reader(out))
hdr, units = rows[0], rows[1]
res = []
for r in rows[2:]:
    d = {}
    for i, h in enumerate(hdr):
        if h in WANT:
            d[h] = r[i] + (" " + units[i] if units[i] else "")
    try:
        rd = float(r[hdr.index("dram__bytes_read.sum")].replace(",", ""))
        wr = float(r[hdr.index("dram__bytes_write.sum")].replace(",", ""))
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
        d["dram_bytes_per_launch"] = int(rd * scale.get(units[hdr.index("dram__bytes_read.sum")], 1) + wr * scale.get(units[hdr.index("dram__bytes_write.sum")], 1))
    except Exception:
        pass
    res.append(d)
print(json.dumps(res, indent=1))
