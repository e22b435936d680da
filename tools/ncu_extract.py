"""Summarise an `ncu --set full` report: python tools/ncu_extract.py report.ncu-rep > summary.txt"""
import csv, subprocess, sys, io
WANT = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'dram__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size', 'launch__shared_mem_per_block_static',
        'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'lts__t_sector_hit_rate.pct', 'l1tex__t_sector_hit_rate.pct',
        'smsp__inst_executed.sum', 'smsp__cycles_active.avg', 'sm__cycles_elapsed.max',
        'smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio', 'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_wait_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_membar_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_drain_per_issue_active.ratio',
        'local_load_bytes', 'smsp__inst_executed_op_local_ld.sum', 'smsp__inst_executed_op_local_st.sum']
out = subprocess.run(['ncu', '-i', sys.argv[1], '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
hdr, units = rows[0], rows[1]
print(f"# ncu --set full --clock-control none; extracted from {sys.argv[1].split('/')[-1]} (cold-cache, serialised replay)")
for r in rows[2:]:
    print(f"\n== {r[hdr.index('Kernel Name')]}  grid {r[hdr.index('launch__grid_size')]} x {r[hdr.index('launch__block_size')]}")
    for w in WANT:
        if w in hdr:
            i = hdr.index(w)
            print(f"  {w:95s} {r[i]:>16s} {units[i]}")
