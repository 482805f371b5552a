#!/usr/bin/env python3
"""One line per profiled launch of an .ncu-rep (run where ncu is installed; no GPU needed):
    python scripts/ncu_summary.py layer_kernels.ncu-rep > layer_kernels.summary.txt
Columns: duration, DRAM bytes read / written, achieved DRAM GB/s, tensor-pipe active %, issue-slot %, warps active %,
registers, grid, and the kernel name."""
import csv
import io
import re
import subprocess
import sys

KEYS = {
    "gpu__time_duration.sum": "dur",
    "dram__bytes_read.sum": "rd",
    "dram__bytes_write.sum": "wr",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor",
    "smsp__issue_active.avg.pct_of_peak_sustained_active": "issue",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "warps",
    "launch__registers_per_thread": "regs",
    "launch__grid_size": "grid",
    "sm__cycles_elapsed.max": "cyc",
    "lts__t_bytes.sum": "l2",
}
UNIT = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "nsecond": 1e-3, "usecond": 1.0, "msecond": 1e3, "ns": 1e-3, "us": 1.0,
        "ms": 1e3}

raw = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, data = rows[0], rows[1], rows[2:]
col = {h: i for i, h in enumerate(hdr)}
print(f"{'us':>8} {'dram rd MB':>10} {'dram wr MB':>10} {'GB/s':>7} {'L2 MB':>8} {'tensor%':>8} {'issue%':>7} {'warps%':>7} {'regs':>5} {'grid':>6}  kernel")
for r in data:
    v = {}
    for k, short in KEYS.items():
        if k in col:
            try:
                x = float(r[col[k]].replace(",", ""))
            except ValueError:
                x = float("nan")
            v[short] = x * UNIT.get(units[col[k]], 1.0)
        else:
            v[short] = float("nan")
    name = re.sub(r"\(.*", "", r[col["Kernel Name"]])
    gbs = (v["rd"] + v["wr"]) / (v["dur"] * 1e-6) / 1e9 if v["dur"] > 0 else float("nan")
    print(f"{v['dur']:8.2f} {v['rd'] / 1e6:10.3f} {v['wr'] / 1e6:10.3f} {gbs:7.0f} {v['l2'] / 1e6:8.2f} {v['tensor']:8.1f} {v['issue']:7.1f} "
          f"{v['warps']:7.1f} {int(v['regs']):5d} {int(v['grid']):6d}  {name}")
