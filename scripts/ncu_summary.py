"""Key numbers of one kernel from an .ncu-rep (ncu --set full): python scripts/ncu_summary.py <rep> > <name>.txt"""
import csv, subprocess, sys, io
rep = sys.argv[1]
raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
want = ['gpu__time_duration.sum', 'launch__grid_size', 'launch__block_size', 'launch__registers_per_thread', 'launch__occupancy_limit_registers',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'smsp__inst_executed.sum', 'sm__inst_executed.avg.per_cycle_elapsed',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'dram__throughput.avg.pct_of_peak_sustained_elapsed',
        'lts__t_sector_hit_rate.pct', 'l1tex__t_sector_hit_rate.pct', 'sm__icc_request_hit_rate.pct', 'smsp__average_warp_latency_per_inst_issued.ratio']
for r in rows[2:]:
    name = r[hdr.index('Kernel Name')] if 'Kernel Name' in hdr else '?'
    print('kernel:', name)
    for h, u, v in zip(hdr, units, r):
        if h in want: print(f'  {h:62s} {v} {u}')
    print('  stall reasons per issued instruction (warps):')
    st = [(float(v or 0), h) for h, v in zip(hdr, r) if h.startswith('smsp__average_warps_issue_stalled_') and h.endswith('_per_issue_active.ratio')]
    for v, h in sorted(st, reverse=True)[:8]: print(f'    {h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]:24s} {v:.2f}')
