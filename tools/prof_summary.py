"""Summarise an ncu --set full report into prof_out/<name>.md (key metrics + hottest source lines); prof_out/ is git-ignored,
copy a summary elsewhere to keep it."""
import csv, os, subprocess, sys
rep, kernel, name = sys.argv[1], sys.argv[2], sys.argv[3]
note = sys.argv[4] if len(sys.argv) > 4 else ""
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv", "--kernel-name", "regex:" + kernel], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units, vals = rows[0], rows[1], rows[2]
d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
keys = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__cycles_elapsed.avg"]
out = ["# %s — ncu summary (`%s`)" % (name, kernel), "", note, "", "Source report: `%s` (ncu --set full --clock-control none --import-source on; under-profiler times are not bench values)." % os.path.basename(rep), "",
       "| metric | value | unit |", "|---|---|---|"]
for k in keys:
    if k in d: out.append("| %s | %s | %s |" % (k, d[k][0], d[k][1]))
out += ["", "Warp stall reasons (average warps stalled per issue-active cycle, > 0.05):", "", "| reason | ratio |", "|---|---|"]
for h, u, v in zip(hdr, units, vals):
    if "average_warps_issue_stalled" in h and h.endswith("_per_issue_active.ratio"):
        try:
            if float(v) > 0.05: out.append("| %s | %s |" % (h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""), v))
        except ValueError: pass
lines = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_lines.py"), rep, kernel], capture_output=True, text=True, env=dict(os.environ, TOP="25")).stdout
out += ["", "Hottest CUDA source lines (warp-stall samples; `-lineinfo`):", "", "```", lines.rstrip(), "```", ""]
os.makedirs(os.path.join(ROOT, "prof_out"), exist_ok=True)
open(os.path.join(ROOT, "prof_out", name + ".md"), "w").write("\n".join(out))
print("wrote prof_out/%s.md" % name)
