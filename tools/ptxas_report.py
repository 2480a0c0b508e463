#!/usr/bin/env python
"""nvcc -Xptxas -v output (stdin or file) -> one line per kernel: registers, stack, spill stores/loads, smem.
   usage: nvcc ... -Xptxas -v ... 2>&1 | python tools/ptxas_report.py [filter-substring]
   The library's sources are graph-neural-networks_b200/build.py's SOURCES: csrc/*.cu, csrc/nv/nv.cu and
   csrc/arma/arma.cu
   (e.g. `... -c graph-neural-networks_b200/csrc/arma/arma.cu ... | python tools/ptxas_report.py arma_`)."""
import re
import subprocess
import sys

txt = sys.stdin.read()
flt = sys.argv[1] if len(sys.argv) > 1 else ""
cur = None
rows = []
for line in txt.splitlines():
    m = re.search(r"Compiling entry function '([^']+)'", line)
    if m:
        cur = {"name": m.group(1)}
        rows.append(cur)
        continue
    if cur is None:
        continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m:
        cur["stack"], cur["sst"], cur["sld"] = map(int, m.groups())
    m = re.search(r"Used (\d+) registers", line)
    if m:
        cur["regs"] = int(m.group(1))
        m2 = re.search(r"(\d+) bytes smem", line)
        cur["smem"] = int(m2.group(1)) if m2 else 0
names = [r["name"] for r in rows]
try:
    dem = subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.splitlines()
except Exception:
    dem = names
for r, d in zip(rows, dem):
    # kernels in an anonymous namespace (csrc/nv/nv.cu, csrc/arma/arma.cu) demangle with "(anonymous namespace)::"
    d = re.sub(r"\(.*", "", d.replace("(anonymous namespace)::", "")).replace("void b200gf::", "").replace("void ", "")
    if flt and flt not in d:
        continue
    print("%-90s regs=%3d stack=%3d spill_st=%3d spill_ld=%3d" % (d[:90], r.get("regs", -1), r.get("stack", -1), r.get("sst", -1), r.get("sld", -1)))
