"""Extract the metrics that matter from `ncu -i X.ncu-rep --page raw --csv` (stdin) -> profiles/<name>_summary.txt."""
import csv
import sys
from pathlib import Path

WANT = ["Kernel Name", "Block Size", "Grid Size", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__waves_per_multiprocessor", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "l1tex__m_xbar2l1tex_read_bytes.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "launch__cluster_size",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem"]
rows = list(csv.reader(sys.stdin))
hdr, units, vals = rows[0], rows[1], rows[2]
(Path(__file__).resolve().parent.parent / "profiles").mkdir(exist_ok=True)
out = open(Path(__file__).resolve().parent.parent / "profiles" / f"{sys.argv[1]}_summary.txt", "w")
for h, u, v in zip(hdr, units, vals):
    if h in WANT:
        line = f"{h} [{u}] = {v}"
        print(line)
        out.write(line + "\n")
