#!/usr/bin/env python
"""Reduce ncu CSV exports to short per-kernel summaries (write them under build/profiles/, which git ignores).
    python tools/ncu_summarize.py raw <ncu --page raw --csv file> <out.csv> "<header comment>"
    python tools/ncu_summarize.py launches <ncu --metrics gpu__time_duration.sum --csv log> <out.csv> "<header comment>"
"""
import csv
import re
import sys
from collections import OrderedDict

KEEP = ['gpu__time_duration.sum', 'sm__cycles_elapsed.max', 'sm__cycles_elapsed.max.per_second',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'sm__inst_executed.sum.per_cycle_elapsed', 'sm__inst_executed.sum',
        'dram__bytes_read.sum', 'dram__bytes_write.sum', 'dram__bytes_read.sum.per_second',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'lts__t_sectors_srcunit_tex_op_read.sum',
        'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum', 'smsp__cycles_active.avg', 'launch__registers_per_thread',
        'launch__shared_mem_per_block_dynamic', 'launch__grid_size', 'launch__cluster_size', 'launch__block_size']


def raw(src, dst, comment):
    rows = list(csv.reader(open(src)))
    hdr = next(i for i, r in enumerate(rows) if r and r[0] == 'ID')
    names, units, vals = rows[hdr], rows[hdr + 1], rows[hdr + 2]
    with open(dst, 'w') as f:
        f.write(f'# {comment}\nmetric,unit,value\n')
        k = names.index('Kernel Name')
        f.write(f'"kernel",,"{vals[k]}"\n')
        for m in KEEP:
            if m in names:
                i = names.index(m)
                f.write(f'{m},{units[i]},{vals[i]}\n')


def launches(src, dst, comment):
    rows = list(csv.reader(l for l in open(src) if not l.startswith('==')))
    hdr = next(i for i, r in enumerate(rows) if r and r[0] == 'ID')
    names = rows[hdr]
    k, v = names.index('Kernel Name'), names.index('Metric Value')
    u = names.index('Metric Unit')
    tot = OrderedDict()
    for r in rows[hdr + 1:]:
        if len(r) <= v:
            continue
        name = re.sub(r'^void |<unnamed>::|\(.*$', '', r[k])
        t = float(r[v].replace(',', ''))
        t = t / 1e3 if r[u] in ('ns', 'nsecond') else (t * 1e3 if r[u] in ('ms', 'msecond') else t)
        n, s = tot.get(name, (0, 0.0))
        tot[name] = (n + 1, s + t)
    total = sum(s for _, s in tot.values())
    with open(dst, 'w') as f:
        f.write(f'# {comment}\nkernel,launches,total_us,share\n')
        for name, (n, s) in sorted(tot.items(), key=lambda kv: -kv[1][1])[:25]:
            f.write(f'"{name}",{n},{s:.1f},{s / total:.4f}\n')


if __name__ == '__main__':
    {'raw': raw, 'launches': launches}[sys.argv[1]](sys.argv[2], sys.argv[3], sys.argv[4])
