"""Where the time of one benchmarked BPR epoch goes, wave by wave.

The epoch is bench.py's: 1M users x 100K items x 50 positives per user, d = 64, fp32, fused Philox sampling with the
rated-set signature pre-test (bpr_epoch_usermajor_sig), then |P|^2 and |Q|^2.  launch_usermajor runs it as waves,
each a snapshot copy of the item table (Q -> Qr, device to device) followed by one user-major kernel launch.

After 3 warm-up epochs, one epoch is traced under torch.profiler (CUDA activities; the trace is written to
OUT/trace.json) and reported as: total epoch time, the Qr copies (sum, median), the user-major launches (sum, median,
min / median / max per wave), the other kernels and the idle gaps between consecutive device activities.  Then,
without the profiler, 20 epochs are timed with CUDA events.  Everything goes to OUT/profile_k1_waves.json as well.

  python tools/profile_k1_waves.py [--out DIR] [--epochs 20]

OUT defaults to a directory under the system's temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

USERS, ITEMS, DEGREE, D = 1_000_000, 100_000, 50, 64
LR, REG = 0.01, 0.001


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
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'qrec_profile_k1_waves'))
    ap.add_argument('--epochs', type=int, default=20)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from qrec_b200 import engine as E
    from qrec_b200 import synthetic
    assert torch.cuda.is_available(), 'profile_k1_waves needs a GPU'
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    on = card()

    data = synthetic.make_interactions(USERS, ITEMS, DEGREE, device=dev)
    P, Q = synthetic.init_tables(USERS, ITEMS, D, seed=1, device=dev)
    rowptr, cols, i = data['sorted_rowptr'], data['sorted_cols'], data['i']
    sig = E.rated_signature(rowptr, cols)
    loss = torch.zeros(3, dtype=torch.float64, device=dev)
    epoch = [0]

    def step():
        E.bpr_epoch_usermajor_sig(P, Q, rowptr, i, rowptr, cols, sig, ITEMS, 2024, epoch[0], LR, REG, REG, loss[0:1])
        E.sumsq(P, loss[1:2])
        E.sumsq(Q, loss[2:3])
        epoch[0] += 1

    for _ in range(3):
        step()
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    trace = os.path.join(args.out, 'trace.json')
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        evs = json.load(f)
    evs = evs['traceEvents'] if isinstance(evs, dict) else evs
    acts = sorted((e for e in evs if e.get('ph') == 'X' and e.get('cat') in ('kernel', 'gpu_memcpy', 'gpu_memset')),
                  key=lambda e: e['ts'])
    assert acts, 'no device activity in the trace'
    is_copy = lambda e: e['cat'] == 'gpu_memcpy' and 'DtoD' in e['name']             # noqa: E731
    is_k1 = lambda e: e['cat'] == 'kernel' and 'bpr_sgd_usermajor' in e['name']       # noqa: E731
    copies = np.array([e['dur'] for e in acts if is_copy(e)])
    k1 = np.array([e['dur'] for e in acts if is_k1(e)])
    other = sum(e['dur'] for e in acts if not (is_copy(e) or is_k1(e)))
    ends = np.array([e['ts'] + e['dur'] for e in acts])
    gaps = np.maximum(np.array([e['ts'] for e in acts[1:]]) - np.maximum.accumulate(ends)[:-1], 0)
    k1_names = sorted({e['name'].replace('(anonymous namespace)::', '').split('(')[0] for e in acts if is_k1(e)})
    prof_rep = {
        'epoch_us': float(ends.max() - acts[0]['ts']),
        'waves': int(len(k1)),
        'qr_copy_us': {'sum': float(copies.sum()), 'median': float(np.median(copies)) if len(copies) else 0.0},
        'k1_us': {'sum': float(k1.sum()), 'median': float(np.median(k1)), 'min': float(k1.min()), 'max': float(k1.max())},
        'other_device_us': float(other),
        'gaps_us': float(gaps.sum()),
        'k1_kernel': k1_names,
    }

    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.epochs):
        step()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.epochs
    rep = {'card': on, 'shape': '%d users x %d items x %d per user, d=%d, signature sampler' % (USERS, ITEMS, DEGREE, D),
           'profiled_epoch': prof_rep,
           'events': {'epochs': args.epochs, 'ms_per_epoch': ms, 'triples_per_s': USERS * DEGREE / (ms * 1e-3)}}
    with open(os.path.join(args.out, 'profile_k1_waves.json'), 'w') as f:
        json.dump(rep, f, indent=1)

    p = prof_rep
    print('card: %s' % on)
    print('one profiled epoch (torch.profiler, CUDA activities), %d waves, kernel %s' % (p['waves'], ', '.join(k1_names)))
    print('  %-28s %10.1f us' % ('epoch, first to last activity', p['epoch_us']))
    print('  %-28s %10.1f us   median %7.1f us' % ('Qr snapshot copies', p['qr_copy_us']['sum'], p['qr_copy_us']['median']))
    print('  %-28s %10.1f us   median %7.1f us   per wave min %.1f / max %.1f us' % (
        'user-major launches', p['k1_us']['sum'], p['k1_us']['median'], p['k1_us']['min'], p['k1_us']['max']))
    print('  %-28s %10.1f us' % ('other kernels and copies', p['other_device_us']))
    print('  %-28s %10.1f us' % ('gaps between activities', p['gaps_us']))
    print('%d epochs, CUDA events, no profiler: %.3f ms per epoch = %.4g triples/s   (%s)' % (
        args.epochs, ms, rep['events']['triples_per_s'], on))


if __name__ == '__main__':
    main()
