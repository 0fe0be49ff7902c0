#!/usr/bin/env python3
"""Summarise an ncu --set full capture of m2s::convert_kernel into profiles/ (markdown + traffic.json).

usage: ncu_summary.py <report.ncu-rep> <layout-name> <out.md>
"""
import csv, json, os, subprocess, sys
rep, layout, out = sys.argv[1:4]
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units, vals = rows[0], rows[1], rows[2]
d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
keys = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.max", "sm__cycles_active.avg",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "lts__t_bytes.sum", "l1tex__t_bytes.sum", "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "smsp__inst_executed_op_global_atom.sum", "smsp__inst_executed_op_global_red.sum"]
kname = d.get("Kernel Name", ("?", ""))[0]
lines = [f"# ncu --set full --clock-control none: {kname}, layout {layout}", "",
         f"source report: {os.path.basename(rep)} (gpurun scratch; numbers below are per launch, cold-cache and serialised by ncu)", "",
         "| metric | value | unit |", "|---|---|---|"]
for k in keys:
    if k in d:
        lines.append(f"| {k} | {d[k][0]} | {d[k][1]} |")
st = []
for h, (v, u) in d.items():
    if "average_warps_issue_stalled" in h and h.endswith("_per_issue_active.ratio"):
        try:
            st.append((float(v), h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", "")))
        except ValueError:
            pass
lines += ["", "## warp stall reasons (average warps stalled per issue-active cycle)", "", "| reason | ratio |", "|---|---|"]
for v, n in sorted(st, reverse=True)[:10]:
    lines.append(f"| {n} | {v:.2f} |")
def num(k):
    v, u = d[k]
    f = float(v)
    return f * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
traffic = num("dram__bytes_read.sum") + num("dram__bytes_write.sum")
lines += ["", f"DRAM traffic per launch: {traffic/1e6:.2f} MB (read {num('dram__bytes_read.sum')/1e6:.2f} + write {num('dram__bytes_write.sum')/1e6:.2f}); "
          "the 126 MB L2 absorbs most of the record writes of one launch, so this is below the algorithmic bytes."]
open(out, "w").write("\n".join(lines) + "\n")
tj = os.path.join(root, "profiles", "traffic.json")
t = json.load(open(tj)) if os.path.exists(tj) else {}
key = layout + ("_raster" if "raster" in kname else "_fragment")
t[key] = traffic
if layout + "_raster" in t and layout + "_fragment" in t:
    t[layout] = t[layout + "_raster"] + t[layout + "_fragment"]  # the whole step = both launches
json.dump(t, open(tj, "w"), indent=1)
print("wrote", out, "traffic", traffic)
