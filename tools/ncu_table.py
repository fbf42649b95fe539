#!/usr/bin/env python
"""One markdown row per kernel launch of an .ncu-rep captured with `ncu --set full`: duration, DRAM bytes, and the
utilisation figures the rooflines quote.  usage: ncu_table.py report.ncu-rep > ncu_<what>.md"""
import csv
import io
import re
import subprocess
import sys

COLS = [("gpu__time_duration.sum", "us", 1.0), ("dram__bytes_read.sum", "DRAM rd MB", None), ("dram__bytes_write.sum", "DRAM wr MB", None),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM %", 1.0),
        ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1 %", 1.0),
        ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %", 1.0),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %", 1.0),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps %", 1.0),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %", 1.0),
        ("smsp__thread_inst_executed_per_inst_executed.ratio", "lanes/inst", 1.0),
        ("smsp__inst_executed.sum", "warp inst (M)", 1e-6), ("launch__registers_per_thread", "regs", 1.0)]
path = sys.argv[1]
out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
print("| # | kernel | grid | " + " | ".join(c[1] for c in COLS) + " |")
print("|---:|---|---|" + "---:|" * len(COLS))
for n, r in enumerate(rows[2:]):
    name = re.sub(r"\(.*", "", r[idx["Kernel Name"]]).replace("void ", "").replace("ffb6d::", "")
    vals = []
    for key, label, mul in COLS:
        if key not in idx or r[idx[key]] in ("", "n/a"):
            vals.append("")
            continue
        v = float(r[idx[key]].replace(",", ""))
        if key == "gpu__time_duration.sum":     # ncu scales the unit per report: normalise to microseconds
            v *= {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "nsecond": 1e-3, "s": 1e6, "second": 1e6}.get(units[idx[key]], 1.0)
            vals.append("%.1f" % v)
        elif mul is None:     # bytes with a unit column
            u = units[idx[key]]
            v *= {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(u, 1.0)
            vals.append("%.2f" % v)
        else:
            vals.append("%.1f" % (v * mul) if abs(v * mul) < 1e5 else "%.0f" % (v * mul))
    print("| %d | `%s` | %s | " % (n, name[:60], r[idx["Grid Size"]]) + " | ".join(vals) + " |")
