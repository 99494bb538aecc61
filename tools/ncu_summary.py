"""Summarise an .ncu-rep (raw page) into a few headline numbers. usage: ncu_summary.py rep [out.md]"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, data = rows[0], rows[1], rows[2:]
want = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__occupancy_limit_registers", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_active", "l1tex__t_sector_hit_rate.pct",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "smsp__average_warp_latency_per_inst_issued.ratio", "smsp__warps_eligible.avg.per_cycle_active",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores"]
stall = [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
lines = []
for k in want + stall:
    if k in hdr:
        i = hdr.index(k)
        vals = [r[i] for r in data]
        if k in stall:
            try:
                if max(float(v) for v in vals) < 0.1:
                    continue
            except ValueError:
                pass
        lines.append("| %s | %s | %s |" % (k, units[i], " / ".join(vals)))
out = "| metric | unit | per captured launch |\n|---|---|---|\n" + "\n".join(lines) + "\n"
if len(sys.argv) > 2:
    open(sys.argv[2], "w").write(out)
print(out)
