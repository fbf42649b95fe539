#!/usr/bin/env python
"""Per-kernel SASS evidence of libffb6d_b200.so: counts of the Hopper-specific opcodes (wgmma -> HGMMA, wgmma
fence / wait -> WARPGROUP, bulk / tensor TMA -> UBLKCP / UTMALDG, mbarrier -> SYNCS, cluster barriers -> UCGABAR,
distributed shared memory -> *.CLUSTER / MAPA), plus LDGSTS / HMMA (legacy paths, expected 0) and the total
instruction count.  usage: sass_summary.py [lib.so] > sass.md   (no GPU needed)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "ffb6d_b200", "libffb6d_b200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
OPS = ["HGMMA", "WARPGROUP", "UBLKCP", "UTMALDG", "UTMASTG", "SYNCS", "UCGABAR", "MAPA",
       "REDUX", "ATOM", "RED", "LDGSTS", "HMMA", "SHFL", "LDS", "STS"]
counts, order, cur = {}, [], None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        name = re.sub(r"\(.*", "", name).replace("void ", "").replace("ffb6d::", "")
        cur = name
        if cur not in counts:
            counts[cur] = collections.Counter()
            order.append(cur)
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1)
        counts[cur]["total"] += 1
        base = op.split(".")[0]
        for o in OPS:
            if base == o or (o in ("ATOM", "RED") and base in (o, o + "G", o + "S")) or (o == "UCGABAR" and base.startswith(o)):
                counts[cur][o] += 1
        if ".CLUSTER" in op or "SHARED::CLUSTER" in op:
            counts[cur]["cluster-scope"] += 1
print("# SASS opcode counts per kernel (`cuobjdump -sass ffb6d_b200/libffb6d_b200.so`, sm_90a)\n")
cols = ["total"] + OPS + ["cluster-scope"]
print("| kernel | " + " | ".join(cols) + " |")
print("|---|" + "---:|" * len(cols))
for k in order:
    if "long long" in k:      # the int64-index twins differ only in the output store
        continue
    c = counts[k]
    print("| `%s` | " % k[:70] + " | ".join(str(c[x]) if c[x] else "" for x in cols) + " |")
