"""Turn an `ncu --set full` report of tools/profile_kernels.py into <prefix>_ncu_summary.{json,md}.
Usage: python tools/ncu_summary.py prof.ncu-rep out/prefix [more.ncu-rep ...]"""
import csv
import io
import json
import re
import subprocess
import sys

W, H = 1920, 1080
METRICS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
           "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
           "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
           "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "smsp__inst_executed.sum",
           "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]


def unit_scale(u):
    return {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1, "us": 1e3, "usecond": 1e3, "nsecond": 1, "msecond": 1e6}.get(u, 1)


def stage_of(name, grid):
    m = re.search(r"rough_search_u8_kernel<(\d)>", name)
    if m:
        return f"rough_search_w{1 << int(m.group(1))}"
    m = re.search(r"intra_recon_kernel<unsigned char, (\d)(?:, (?:false|\(bool\)0), (\d))?>", name)
    if m:
        w = 1 << int(m.group(1))
        g = max(1, 1024 // (w * w))
        luma = -(-((W // w) * (H // w)) // g)
        suffix = "_inv" if m.group(2) == "2" else ""
        if grid == luma:
            return f"recon_luma{suffix}_w{w}"
        return f"recon_chroma{suffix}_w{2 * w}"
    m = re.search(r"rdoq_grid(?:_thread)?_kernel<(\d)", name)
    if m:
        w = 1 << int(m.group(1))
        thread = "thread" in name
        per = 128 if thread else {4: 8, 8: 8, 16: 2, 32: 1}[w]
        luma = -(-((W // w) * (H // w)) // per)
        return f"rdoq_luma_w{w}" if grid == luma else f"rdoq_chroma_w{2 * w}"
    m = re.search(r"deblock_pass_kernel<unsigned char, (?:\(bool\))?(\w+)>", name)
    if m:
        return "deblock_hor" if m.group(1) in ("true", "1") else "deblock_ver"
    m = re.search(r"satd_nxn_kernel<unsigned char, (\d+)>", name)
    if m:
        return f"satd_nxn_kernel_{m.group(1)}"
    if "sao_ctu_kernel" in name:
        return "sao_stats_decide"
    return re.sub(r"\(.*", "", name).split("::")[-1]


def main():
    reps, tag = [sys.argv[1]] + sys.argv[3:], sys.argv[2]
    out = {}
    for rep in reps:
        txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(txt)))
        hdr, units = rows[0], rows[1]
        ki = hdr.index("Kernel Name")
        for row in rows[2:]:
            vals = {}
            for m in METRICS:
                if m in hdr:
                    i = hdr.index(m)
                    try:
                        vals[m] = float(row[i].replace(",", "")) * unit_scale(units[i])
                    except ValueError:
                        pass
            st = stage_of(row[ki], int(vals.get("launch__grid_size", 0)))
            d = out.setdefault(st, {"kernel": re.sub(r"\(.*", "", row[ki]), "launches": 0, "time_ns": 0.0, "dram_read": 0.0, "dram_write": 0.0})
            d["launches"] += 1
            d["time_ns"] += vals.get("gpu__time_duration.sum", 0)
            d["dram_read"] += vals.get("dram__bytes_read.sum", 0)
            d["dram_write"] += vals.get("dram__bytes_write.sum", 0)
            d["grid"] = int(vals.get("launch__grid_size", 0))
            d["block"] = int(vals.get("launch__block_size", 0))
            d["regs"] = int(vals.get("launch__registers_per_thread", 0))
            d["issue_active_pct"] = round(vals.get("smsp__issue_active.avg.pct_of_peak_sustained_active", 0), 1)
            d["sm_throughput_pct"] = round(vals.get("sm__throughput.avg.pct_of_peak_sustained_elapsed", 0), 1)
            d["dram_throughput_pct"] = round(vals.get("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", 0), 1)
            d["warps_active_pct"] = round(vals.get("sm__warps_active.avg.pct_of_peak_sustained_active", 0), 1)
            d["tensor_pipe_pct"] = round(vals.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0), 2)
            d["warp_instructions"] = int(vals.get("smsp__inst_executed.sum", 0))
            d["smem_bank_conflicts"] = int(vals.get("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", 0))
    for st, d in out.items():
        n = d["launches"]
        d["us_per_launch"] = round(d.pop("time_ns") / n / 1e3, 2)
        d["dram_bytes_per_launch"] = int((d.pop("dram_read") + d.pop("dram_write")) / n)
    json.dump(out, open(tag + "_ncu_summary.json", "w"), indent=1, sort_keys=True)
    with open(tag + "_ncu_summary.md", "w") as f:
        f.write("| stage | kernel | grid x block | regs | us/launch (ncu, cold) | DRAM bytes/launch | DRAM % | SM % | issue-active % | warps-active % | tensor pipe % |\n|---|---|---|---|---|---|---|---|---|---|---|\n")
        for st, d in sorted(out.items(), key=lambda kv: -kv[1]["us_per_launch"]):
            f.write(f"| {st} | `{d['kernel'].split('::')[-1]}` | {d['grid']} x {d['block']} | {d['regs']} | {d['us_per_launch']} | {d['dram_bytes_per_launch']:,} | "
                    f"{d['dram_throughput_pct']} | {d['sm_throughput_pct']} | {d['issue_active_pct']} | {d['warps_active_pct']} | {d['tensor_pipe_pct']} |\n")
    print(open(tag + "_ncu_summary.md").read())


if __name__ == "__main__":
    main()
