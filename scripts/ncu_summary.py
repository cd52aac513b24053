"""Summarise an `ncu --set full` report (any kernels) into a text summary: per launch the duration, DRAM bytes,
DRAM / tensor / issue utilisation, occupancy, registers, grid.   python scripts/ncu_summary.py report.ncu-rep [note]"""
import csv
import subprocess
import sys

rep = sys.argv[1]
note = sys.argv[2] if len(sys.argv) > 2 else ""
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
keys = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__waves_per_multiprocessor"]
ik = hdr.index("Kernel Name")
for r in rows[2:]:
    print(f"== {r[ik][:90]}  ({note})")
    for k in keys:
        if k in hdr:
            i = hdr.index(k)
            print(f"  {k:75s} {r[i]} {units[i]}")
