"""Summarise an .ncu-rep (read here, no GPU needed) into a small markdown table for profiles/.
usage: python tools/ncu_summary.py x.ncu-rep [kernel-regex] > x.md"""
import csv
import io
import re
import subprocess
import sys

KEYS = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'lts__throughput.avg.pct_of_peak_sustained_elapsed', 'l1tex__throughput.avg.pct_of_peak_sustained_elapsed',
        'l1tex__t_sector_hit_rate.pct', 'lts__t_sector_hit_rate.pct',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tensor.sum', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size',
        'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_registers', 'launch__waves_per_multiprocessor']


def main():
    rep = sys.argv[1]
    pat = re.compile(sys.argv[2]) if len(sys.argv) > 2 else None
    out = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    print('# ncu summary: %s\n' % rep)
    for r in rows[2:]:
        name = r[idx['Kernel Name']]
        if pat and not pat.search(name):
            continue
        print('## %s  (id %s)\n' % (name[:120], r[idx.get('ID', 0)]))
        print('| metric | value | unit |\n|---|---|---|')
        for k in KEYS:
            if k in idx:
                print('| %s | %s | %s |' % (k, r[idx[k]], units[idx[k]]))
        print()


if __name__ == '__main__':
    main()
