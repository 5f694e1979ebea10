#!/usr/bin/env python
"""Condenses `ncu -i X.ncu-rep --page raw --csv` exports into a handful of summary numbers.
    python tools/ncu_summary.py gpurun_out/r2/*_raw.csv [--json out.json]"""
import csv
import json
import sys

KEYS = [('ms', 'gpu__time_duration.sum', 1e-6), ('dram_read_GB', 'dram__bytes_read.sum', 1e-9), ('dram_write_GB', 'dram__bytes_write.sum', 1e-9),
        ('dram_pct', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 1), ('l2_hit_pct', 'lts__t_sector_hit_rate.pct', 1),
        ('lts_pct', 'lts__throughput.avg.pct_of_peak_sustained_elapsed', 1), ('l1tex_pct', 'l1tex__throughput.avg.pct_of_peak_sustained_elapsed', 1),
        ('sm_pct', 'sm__throughput.avg.pct_of_peak_sustained_elapsed', 1), ('lts_atomic_pct', 'lts__d_atomic_input_cycles_active.avg.pct_of_peak_sustained_elapsed', 1),
        ('warps_active_pct', 'sm__warps_active.avg.pct_of_peak_sustained_active', 1), ('regs', 'launch__registers_per_thread', 1),
        ('grid', 'launch__grid_size', 1), ('red_sectors', 'l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum', 1)]


def num(x):
    try:
        return float(str(x).replace(',', ''))
    except ValueError:
        return None


def main():
    out = {}
    paths = [a for a in sys.argv[1:] if not a.startswith('--')]
    for path in paths:
        rows = list(csv.reader(open(path)))
        if len(rows) < 3:
            continue
        head, units = rows[0], rows[1]
        ix = {k: n for n, k in enumerate(head)}
        for r in rows[2:]:
            name = r[ix['Kernel Name']][:70]
            rec = {}
            for short, col, scale in KEYS:
                if col in ix:
                    v = num(r[ix[col]])
                    if v is None:
                        continue
                    u = units[ix[col]]
                    if short == 'ms':                      # the raw page reports ns / us / ms depending on the value
                        v = v * {'ns': 1e-6, 'us': 1e-3, 'usecond': 1e-3, 'ms': 1.0, 'msecond': 1.0, 'nsecond': 1e-6, 's': 1e3, 'second': 1e3}.get(u, 1e-6)
                    elif short.startswith('dram_') and short.endswith('GB'):
                        v = v * {'byte': 1e-9, 'Kbyte': 1e-6, 'Mbyte': 1e-3, 'Gbyte': 1.0}.get(u, 1e-9)
                    rec[short] = round(v, 4)
            out.setdefault(path.split('/')[-1], []).append({'kernel': name, **rec})
    print(json.dumps(out, indent=1))
    if '--json' in sys.argv:
        json.dump(out, open(sys.argv[sys.argv.index('--json') + 1], 'w'), indent=1)


if __name__ == '__main__':
    main()
