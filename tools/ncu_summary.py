#!/usr/bin/env python3
"""Developer tool: the metrics of an ncu report that DESIGN.md discusses, one block per kernel.

  python tools/ncu_summary.py <report>.ncu-rep [--json out.json]

--json writes {"dram_bytes_per_search": read + written bytes summed over the kernels of the report, ...} (the
`roofline.traffic` of bench.py)."""
import csv
import json
import subprocess
import sys

WANT = ['gpu__time_duration.sum', 'launch__grid_size', 'launch__block_size', 'launch__registers_per_thread',
        'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem',
        'smsp__inst_executed.sum', 'smsp__thread_inst_executed_per_inst_executed.ratio',
        'smsp__issue_active.avg.per_cycle_active', 'sm__warps_active.avg.per_cycle_active',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__icc_request_hit_rate.pct', 'l1tex__t_sector_hit_rate.pct', 'lts__t_sector_hit_rate.pct',
        'dram__bytes_read.sum', 'dram__bytes_write.sum', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'sass__inst_executed_local_loads', 'sass__inst_executed_local_stores', 'sass__inst_executed_shared_loads',
        'sass__inst_executed_shared_stores', 'sass__inst_executed_global_loads', 'sass__inst_executed_global_stores']
UNIT = {'byte': 1, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9, 'Tbyte': 1e12}


def main():
    rep = sys.argv[1]
    out_json = sys.argv[sys.argv.index('--json') + 1] if '--json' in sys.argv else None
    txt = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    hdr, units = rows[0], rows[1]
    total = 0.0
    per_kernel = {}
    for r in rows[2:]:
        name = r[hdr.index('Kernel Name')]
        short = name.split('(')[0].replace('void ', '').replace('metis::', '')
        print(f'== {short}')
        traffic = 0.0
        for i, h in enumerate(hdr):
            if h in WANT or ('issue_stalled' in h and h.endswith('per_issue_active.ratio')):
                print(f'{h} {units[i]} {r[i]}')
            if h in ('dram__bytes_read.sum', 'dram__bytes_write.sum'):
                traffic += float(r[i]) * UNIT.get(units[i], 1)
        per_kernel[short] = per_kernel.get(short, 0) + int(traffic)
        total += traffic
        print()
    if out_json:
        json.dump({'dram_bytes_per_search': int(total), 'per_kernel': per_kernel,
                   'source': f'ncu --set full --clock-control none, {rep.split("/")[-1]}: dram__bytes_read.sum + '
                             f'dram__bytes_write.sum of the evaluation kernels of one search (bulk round + chain kernel)'},
                  open(out_json, 'w'), indent=1)


if __name__ == '__main__':
    main()
