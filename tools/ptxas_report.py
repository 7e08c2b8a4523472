#!/usr/bin/env python
"""Compile csrc/engine.cu with -Xptxas -v (no GPU needed) and print registers / spills / static smem per kernel."""
import re
import subprocess
import sys

src = sys.argv[1] if len(sys.argv) > 1 else "bert_vits2_b200/csrc/engine.cu"
extra = sys.argv[2:]
cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v",
       "-o", "/tmp/ptxas_report.so", src] + extra
out = subprocess.run(cmd, capture_output=True, text=True).stderr
cur = None
rows = []
for line in out.splitlines():
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m:
        cur = {"name": subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip(), "spill": "0/0"}
        rows.append(cur)
        continue
    if cur is None:
        if "error" in line:
            print(line)
        continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m and "stack" not in cur:
        cur["stack"] = m.group(1); cur["spill"] = f"{m.group(2)}/{m.group(3)}"
    m = re.search(r"Used (\d+) registers", line)
    if m:
        cur["regs"] = m.group(1)
for r in rows:
    n = re.sub(r"\(.*", "", r["name"]).replace("void bv2::", "")
    print(f"{n:60s} regs {r.get('regs','?'):>4s}  stack {r.get('stack','0'):>4s}  spill st/ld {r['spill']}")
if "error" in out:
    print(out[-3000:])
