"""How much of the L2-resident row-op rate the user-major BPR epoch's working set can keep.

The benchmarked epoch (bench.py: 100K items, d = 64) gathers item rows from the wave's snapshot Qr and scatter-adds
into Q: two 25.6 MB tables, 51.2 MB together, against the H100's 50 MB L2.  This runs csrc/microbench.cu
(ubench_row_ops: random 256-byte row gathers, scatter-adds, and one of each) on tables of 100K rows (Q alone),
200K rows (the Q + Qr working set) and 400K rows (twice that), and reports each rate next to the 100K one.

  python tools/probe_k1_l2.py [--ops 200000000] [--out DIR]

The card's name and power limit are printed with the numbers; the JSON goes to OUT/probe_k1_l2.json.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROWS = (100_000, 200_000, 400_000)
MODES = ((0, 'gather', 1), (1, 'scatter_add', 1), (2, 'gather_plus_scatter_add', 2))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '-i', os.environ.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0],
                            '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q or 'unknown card'
    except (OSError, subprocess.SubprocessError):
        return 'unknown card'


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--ops', type=int, default=200_000_000, help='row operations per timed launch')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'qrec_probe_k1_l2'))
    args = ap.parse_args()
    import torch
    from qrec_b200 import engine as E
    assert torch.cuda.is_available(), 'probe_k1_l2 needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    on = card()
    res = {}
    for rows in ROWS:
        T = torch.rand(rows, 64, device=dev)
        sec = {}
        for mode, label, rows_per_op in MODES:
            E.ubench_row_ops(T, args.ops // 10, mode)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                E.ubench_row_ops(T, args.ops, mode)
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / args.reps
            sec[label] = {'ops_per_s': args.ops / (ms * 1e-3), 'GBs': args.ops * rows_per_op * 256 / (ms * 1e-3) / 1e9, 'ms': ms}
        res[rows] = sec
        del T
    base = res[ROWS[0]]
    print('card: %s' % on)
    print('%-10s %-8s %-26s %14s %10s %12s' % ('rows', 'MB', 'op', 'ops/s', 'GB/s', 'vs 100K rows'))
    for rows in ROWS:
        for _, label, _ in MODES:
            r = res[rows][label]
            r['frac_of_100K_rate'] = r['ops_per_s'] / base[label]['ops_per_s']
            print('%-10d %-8.1f %-26s %14.4g %10.1f %12.3f   (%s)' % (rows, rows * 256 / 1e6, label, r['ops_per_s'], r['GBs'],
                                                                  r['frac_of_100K_rate'], on))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'probe_k1_l2.json'), 'w') as f:
        json.dump({'card': on, 'ops_per_launch': args.ops, 'rates': {str(k): v for k, v in res.items()}}, f, indent=1)


if __name__ == '__main__':
    main()
