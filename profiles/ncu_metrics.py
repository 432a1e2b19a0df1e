#!/usr/bin/env python
"""Prints the headline metrics of an .ncu-rep (run where ncu is installed; no GPU needed):
    python profiles/ncu_metrics.py prof.ncu-rep"""
import csv
import subprocess
import sys

WANT = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'launch__registers_per_thread',
        'launch__grid_size', 'launch__block_size', 'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'l1tex__t_sector_hit_rate.pct', 'lts__t_sector_hit_rate.pct',
        'smsp__inst_executed.sum', 'smsp__cycles_active.avg', 'sm__cycles_elapsed.max',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum', 'l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum',
        'l1tex__data_pipe_lsu_wavefronts.sum', 'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum',
        'l1tex__throughput.avg.pct_of_peak_sustained_elapsed', 'lts__throughput.avg.pct_of_peak_sustained_elapsed',
        'smsp__thread_inst_executed_per_inst_executed.ratio', 'l1tex__m_xbar2l1tex_read_bytes.sum',
        'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_wait_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio',
        'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active',
        'smsp__inst_executed_op_shared_ld.sum', 'smsp__inst_executed_op_global_ld.sum', 'smsp__inst_executed_op_global_st.sum']


def main():
    rep = sys.argv[1]
    out = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr = rows[0]
    ki = hdr.index('Kernel Name')
    print('kernels:', [r[ki][:50] for r in rows[2:]])
    for w in WANT:
        if w in hdr:
            i = hdr.index(w)
            print(f'{w:85s} {rows[1][i]:>14s} ', [r[i] for r in rows[2:]])
    if len(sys.argv) > 2:
        for w in hdr:
            if sys.argv[2] in w:
                i = hdr.index(w)
                print(f'{w:85s} {rows[1][i]:>14s} ', [r[i] for r in rows[2:]])


if __name__ == '__main__':
    main()
