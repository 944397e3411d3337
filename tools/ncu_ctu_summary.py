#!/usr/bin/env python
"""Summary of an `ncu --set full --import-source on` capture of ctu_frame_kernel: key metrics, executed warp instructions
and stall samples per device function (SASS ranges from nvdisasm of the object that was profiled).

    python tools/ncu_ctu_summary.py ctu_frame_1080p_medium.ncu-rep build/obj/ctu_driver.o "title" > summary.md
"""
import csv
import io
import os
import re
import subprocess
import sys
import tempfile


def run(cmd, **kw):
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, **kw).stdout


def function_of_each_instruction(obj):
    with tempfile.TemporaryDirectory() as d:
        subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=d, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        cubin = [f for f in os.listdir(d) if f.endswith(".cubin")][0]
        dis = run(["nvdisasm", "-c", os.path.join(d, cubin)])
    names, cur, infn = [], "kernel body", False
    for ln in dis.splitlines():
        if ln.startswith("_ZN") and "ctu_frame_kernel" in ln:
            infn, cur = True, "kernel body"
            continue
        if ln.startswith("_ZN") and "ctu_frame_kernel" not in ln:
            infn = False
        if ln.startswith("$_ZN") and "ctu_frame_kernel" in ln:
            infn = True
            m = re.search(r"\$_ZN6kvzctu\d+([A-Za-z_0-9]+?)(ILi\d+EE)?E", ln)
            cur = (m.group(1) + (m.group(2) or "")) if m else "?"
            continue
        if ln.startswith("$_ZN") and "ctu_frame_kernel" not in ln:
            infn = False
        if infn and re.match(r"\s+/\*[0-9a-f]{4,}\*/", ln):
            names.append(cur)
    return names


def main():
    rep, obj, title = sys.argv[1], sys.argv[2], sys.argv[3]
    raw = list(csv.reader(io.StringIO(run(["ncu", "-i", rep, "--page", "raw", "--csv"]))))
    hdr, units, vals = raw[0], raw[1], raw[2]
    get = lambda n: next(((vals[i], units[i]) for i, h in enumerate(hdr) if h == n), ("n/a", ""))
    print(f"# {title}\n")
    print("| metric | value |\n|---|---|")
    for m in ("gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__occupancy_limit_shared_mem",
              "launch__occupancy_limit_registers", "smsp__inst_executed.sum", "sm__inst_executed.avg.per_cycle_active",
              "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
              "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
              "dram__bytes_read.sum", "dram__bytes_write.sum"):
        v, u = get(m)
        print(f"| {m} | {v} {u} |")
    src = list(csv.reader(io.StringIO(run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"]))))
    h2, data = src[1], src[2:]
    names = function_of_each_instruction(obj)
    if len(names) != len(data):
        print(f"\n(warning: {len(names)} instructions in the object, {len(data)} in the report: per-function attribution skipped)")
        return
    ie, ss = h2.index("Instructions Executed"), h2.index("# Samples")
    cols = {k: h2.index(k) for k in ("stall_barrier", "stall_long_sb", "stall_wait", "stall_no_inst", "stall_selected", "stall_branch_resolving",
                                     "stall_short_sb", "stall_sleep")}
    agg = {}
    for i, r in enumerate(data):
        a = agg.setdefault(names[i], dict(inst=0, samples=0, **{k: 0 for k in cols}))
        a["inst"] += int(r[ie] or 0)
        a["samples"] += int(r[ss] or 0)
        for k, c in cols.items():
            a[k] += int(r[c] or 0)
    ti, ts = sum(a["inst"] for a in agg.values()), sum(a["samples"] for a in agg.values())
    print("\n## Executed warp instructions and stall samples by function\n")
    print("| function | warp instr | % | samples | % | barrier | long_sb | wait | no_inst | selected |\n|---|---|---|---|---|---|---|---|---|---|")
    for n, a in sorted(agg.items(), key=lambda kv: -kv[1]["inst"])[:26]:
        print(f"| {n} | {a['inst']} | {100 * a['inst'] / ti:.1f} | {a['samples']} | {100 * a['samples'] / ts:.1f} | {a['stall_barrier']} | {a['stall_long_sb']} | "
              f"{a['stall_wait']} | {a['stall_no_inst']} | {a['stall_selected']} |")
    tot = {k: sum(a[k] for a in agg.values()) for k in cols}
    print("\nStall totals (all warps): " + ", ".join(f"{k} {v}" for k, v in sorted(tot.items(), key=lambda kv: -kv[1])))
    print(f"\nTotal executed warp instructions: {ti} ({ti / 510:.0f} per CTU at 1080p).")


if __name__ == "__main__":
    main()
