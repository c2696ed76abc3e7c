"""Summarise an .ncu-rep (raw page) into the handful of numbers a kernel review quotes."""
import csv, subprocess, sys
rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr = rows[0]
units = dict(zip(rows[0], rows[1]))
want = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.sum",
        "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
        "sm__cycles_active.avg", "sm__inst_executed_pipe_alu.sum", "sm__inst_executed_pipe_fma.sum", "sm__inst_executed_pipe_xu.sum",
        "sm__inst_executed_pipe_lsu.sum", "sm__inst_executed_pipe_cbu.sum", "sm__inst_executed_pipe_adu.sum", "sm__inst_executed_pipe_uniform.sum"]
for r in rows[2:]:
    d = dict(zip(hdr, r))
    for w in want:
        if w in d:
            print(f"{w} = {d[w]} {units.get(w, '')}".rstrip())
    print("----")
