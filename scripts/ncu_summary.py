"""Summarise an .ncu-rep (read here, no GPU) into a small text file."""
import csv, subprocess, sys, io
rep, out = sys.argv[1], sys.argv[2]
raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
KEYS = ['Kernel Name', 'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'lts__t_bytes.sum', 'lts__throughput.avg.pct_of_peak_sustained_elapsed',
        'l1tex__throughput.avg.pct_of_peak_sustained_elapsed',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tensor.sum', 'smsp__inst_executed.sum', 'sm__cycles_elapsed.max',
        'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size',
        'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_shared_mem',
        'launch__occupancy_limit_registers', 'l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum',
        'l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'smsp__issue_active.avg.pct_of_peak_sustained_active']
STALL = 'smsp__average_warps_issue_stalled_'
with open(out, 'w') as f:
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        f.write('== launch %s ==\n' % d.get('ID', '?'))
        for k in KEYS:
            if k in d:
                f.write(f'{k:75s} {d[k]} {units[hdr.index(k)]}\n')
        st = sorted(((float(v or 0), h) for h, v in d.items() if h.startswith(STALL) and h.endswith('per_issue_active.ratio')), reverse=True)[:8]
        for v, h in st:
            f.write(f'  stall {h[len(STALL):-len("_per_issue_active.ratio")]:40s} {v:.3f} warps/issue\n')
print(open(out).read())
