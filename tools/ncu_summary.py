"""Extracts the metrics the roofline discussion uses from an .ncu-rep (run here, no GPU needed):
   python tools/ncu_summary.py prof.ncu-rep > summary.txt"""
import csv
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__grid_size", "launch__block_size",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed.avg.per_cycle_active", "smsp__inst_executed.sum",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sass__inst_executed_register_spilling", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "sm__cycles_elapsed.max", "sm__cycles_elapsed.max.per_second"]

rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
H, U = rows[0], rows[1]
for r in rows[2:]:
    name = r[H.index("Kernel Name")]
    print(f"# kernel: {name}")
    for k in KEYS:
        if k in H:
            i = H.index(k)
            print(f"{k:95s} {r[i]:>20s} {U[i]}")
    print()
