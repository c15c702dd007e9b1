#!/usr/bin/env python
"""Summarises an `ncu --set full --import-source on` report of dcsim_advance_kernel into a small markdown file.

    python profiles/summarize_ncu.py advance.ncu-rep <events_in_the_profiled_launch> > advance_ncu.md
"""
import collections
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "sm__cycles_elapsed.avg", "sm__cycles_elapsed.avg.per_second",
    "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "launch__waves_per_multiprocessor", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__warps_active.avg.per_cycle_active", "smsp__warps_eligible.avg.per_cycle_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed.avg.per_cycle_elapsed",
    "sm__inst_executed.sum.per_cycle_elapsed", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "sass__inst_executed_local_loads", "sass__inst_executed_local_stores",
]


def ncu(rep, *args):
    return subprocess.run(["ncu", "-i", rep, *args], capture_output=True, text=True).stdout


def main():
    rep, events = sys.argv[1], float(sys.argv[2])
    rows = list(csv.reader(io.StringIO(ncu(rep, "--page", "raw", "--csv"))))
    hdr, units, vals = rows[0], rows[1], rows[2]
    m = {h: (vals[i], units[i]) for i, h in enumerate(hdr)}
    kname = m.get("Kernel Name", ("?", ""))[0].split("(")[0].replace("void ", "")
    print(f"# ncu summary of `{rep.split('/')[-1]}` — `{kname}`, {events:.0f} events in the profiled launch\n")
    print("| metric | value | unit |\n|---|---|---|")
    for k in KEYS:
        if k in m:
            print(f"| `{k}` | {m[k][0]} | {m[k][1]} |")
    stall = {h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""): float(v[0])
             for h, v in m.items() if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio") and v[0]}
    if stall:
        print("\n## warp stall reasons (average warps stalled per issue-active cycle)\n")
        for h, v in sorted(stall.items(), key=lambda kv: -kv[1])[:10]:
            print(f"* {h}: {v:.2f}")

    rows = list(csv.reader(io.StringIO(ncu(rep, "--page", "source", "--csv", "--print-source", "cuda,sass"))))
    agg = collections.defaultdict(lambda: [0, 0, ""])
    cur = None
    col = {}
    for r in rows:
        if not r:
            continue
        if r[0] == "File Path":
            cur = r[1].split("/")[-1]
        elif r[0] == "Line No":
            col = {name: i for i, name in enumerate(r)}
        elif r[0] not in ("", "Function Name"):
            try:
                line = int(r[0])
            except ValueError:
                continue
            def g(name):
                try:
                    return int(r[col[name]].replace(",", ""))
                except (KeyError, IndexError, ValueError):  # a source line with commas and quotes shifts the row
                    return 0
            a = agg[(cur, line)]
            a[0] += g("Instructions Executed")
            a[1] += g("Warp Stall Sampling (All Samples)")
            a[2] = r[1].strip()[:100]
    ti = sum(v[0] for v in agg.values()) or 1
    ts = sum(v[1] for v in agg.values()) or 1
    # The source page lists an instruction once per source FILE of its inline stack (callee line, wrapper line, call
    # site), so summing its rows counts inlined code several times (round 1's "303 per event" was that sum; the same
    # report's sm__inst_executed gave 235).  The per-event figure therefore comes from the hardware counter:
    try:
        cyc = float(m["sm__cycles_elapsed.avg"][0].replace(",", ""))
        ipc = float(m["sm__inst_executed.sum.per_cycle_elapsed"][0].replace(",", ""))
        executed = cyc * ipc
    except (KeyError, ValueError):
        executed = float("nan")
    print(f"\n## per-event cost\n\n* warp-instructions executed (`sm__inst_executed.sum` = sum.per_cycle_elapsed x cycles): "
          f"{executed:.4g} = **{executed / events:.0f} per event**")
    print(f"* (sum over the source page's line rows, which repeats inlined instructions once per file of the inline stack: "
          f"{ti / events:.0f} per event — the table below is INCLUSIVE in that sense; percentages are of this sum)")
    if "dram__bytes_read.sum" in m:
        print(f"* DRAM bytes (read+write) as reported above; algorithmic bytes per event = 96 + 76*D")
    print("\n## top source lines by executed warp-instructions\n\n| file:line | instr/event | % instr | % stall samples | source |\n|---|---|---|---|---|")
    for (f, ln), v in sorted(agg.items(), key=lambda kv: -kv[1][0])[:30]:
        print(f"| {f}:{ln} | {v[0] / events:.1f} | {100 * v[0] / ti:.1f} | {100 * v[1] / ts:.1f} | `{v[2]}` |")


if __name__ == "__main__":
    main()
