#!/usr/bin/env python
"""Summarises .ncu-rep captures (key metrics per kernel)."""
import csv, subprocess, sys
WANT = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'l1tex__throughput.avg.pct_of_peak_sustained_elapsed', 'lts__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread',
        'launch__occupancy_limit_shared_mem', 'launch__occupancy_limit_registers', 'smsp__inst_executed.sum',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum',
        'l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'l1tex__t_sector_hit_rate.pct', 'lts__t_sector_hit_rate.pct', 'sm__inst_executed_pipe_fp64.sum',
        'sm__inst_executed_pipe_xu.sum', 'sm__inst_executed_pipe_lsu.sum', 'sm__inst_executed_pipe_alu.sum',
        'sm__inst_executed_pipe_fma.sum', 'smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio',
        'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_wait_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio']
for rep in sys.argv[1:]:
    out = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    H, U = rows[0], rows[1]
    for r in rows[2:]:
        print(f"== {rep} :: {r[H.index('Kernel Name')][:60]} grid={r[H.index('Grid Size')]} block={r[H.index('Block Size')]}")
        for w in WANT:
            if w in H:
                i = H.index(w)
                print(f"   {w:78s} {r[i]:>18s} {U[i]}")
