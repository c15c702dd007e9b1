#!/usr/bin/env python
"""Where the local-memory traffic (register spills) of a kernel is: LDL/STL instructions of an ncu report with their
executed counts, the source line each belongs to, and the hot SASS neighbourhood.

    python tools/ncu_spills.py x.ncu-rep <events>
"""
import csv
import io
import subprocess
import sys

rep, events = sys.argv[1], float(sys.argv[2])
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
# Every SASS instruction is listed once per source file of its inline stack: de-duplicate by address and remember all
# the source lines it was listed under (innermost callee ... call site).
col, cur_line, seen = {}, "", {}
for r in rows:
    if not r:
        continue
    if r[0] == "Line No":
        col = {name: i for i, name in enumerate(r)}
        continue
    if not col or len(r) <= col["Instructions Executed"]:
        continue
    if r[0] not in ("", "File Path", "Function Name"):          # a CUDA source line row
        cur_line = (r[0] + ": " + r[1]).strip()[:110]
        continue
    if not r[2].startswith("0x"):
        continue
    try:
        n = float(r[col["Instructions Executed"]] or 0)
    except ValueError:
        continue
    e = seen.setdefault(r[2], {"sass": r[3].strip(), "n": n, "lines": []})
    e["lines"].append(cur_line)
tot_all = sum(e["n"] for e in seen.values())
agg, tot = {}, 0.0
for e in seen.values():
    parts = e["sass"].split()
    op = parts[1] if parts and parts[0].startswith("@") and len(parts) > 1 else (parts[0] if parts else "")
    if op.startswith(("LDL", "STL")):
        k = (" <- ".join(e["lines"][:3]), op.split(".")[0])
        agg[k] = agg.get(k, 0.0) + e["n"]
        tot += e["n"]
print(f"executed warp-instructions (unique SASS addresses): {tot_all / events:.1f} per event; local-memory instructions: {tot / events:.2f} per event")
for (line, op), n in sorted(agg.items(), key=lambda kv: -kv[1])[:30]:
    print(f"{n / events:6.2f}  {op:4s} {line}")
