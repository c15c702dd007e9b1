#!/usr/bin/env python
"""Per-opcode breakdown of the executed warp-instructions of a profiled kernel (ncu --set full --import-source on).

    python profiles/opcode_histogram.py advance.ncu-rep <events_in_the_profiled_launch>
"""
import collections
import csv
import io
import subprocess
import sys

rep, events = sys.argv[1], float(sys.argv[2])
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
hdr = next(r for r in rows if r and r[0] == "Address")
col = {n: i for i, n in enumerate(hdr)}
ops = collections.defaultdict(lambda: [0, 0, 0, 0])   # executed, thread-instr, stall samples, static count
for r in rows:
    if not r or not r[0].startswith("0x"):
        continue
    text = r[col["Source"]].strip()
    toks = text.split()
    op = toks[1] if toks[0].startswith("@") and len(toks) > 1 else toks[0]
    op = op.rstrip(";")
    base = op.split(".")[0]
    ex = int(r[col["Instructions Executed"]] or 0)
    a = ops[base]
    a[0] += ex
    a[1] += int(r[col["Thread Instructions Executed"]] or 0)
    a[2] += int(r[col["Warp Stall Sampling (All Samples)"]] or 0)
    a[3] += 1
tot = sum(v[0] for v in ops.values()) or 1
tots = sum(v[2] for v in ops.values()) or 1
print(f"# executed warp-instructions by opcode — `{rep.split('/')[-1]}`, {events:.0f} events, {tot / events:.0f} instr/event\n")
print("| opcode | instr/event | % of executed | avg active lanes | % of stall samples | static count |\n|---|---|---|---|---|---|")
for op, v in sorted(ops.items(), key=lambda kv: -kv[1][0])[:40]:
    if v[0] == 0:
        continue
    print(f"| `{op}` | {v[0] / events:.1f} | {100 * v[0] / tot:.1f} | {v[1] / v[0]:.1f} | {100 * v[2] / tots:.1f} | {v[3]} |")
