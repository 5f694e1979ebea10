#!/usr/bin/env python
"""K11 (SVD++) timings.  One JSON line per measurement, each with the card's name and power limit read in the same
run.

  * parity: one FilmTrust epoch (33 750 entries, d = 10, the golden fixture's tables and first visiting order) through
    qrec_svdpp_sgd_ordered_f64 and _f32, timed with CUDA events after a warm-up epoch, against one epoch of the numpy
    oracle's literal loop (oracle/svdpp_oracle.py) on this host's CPU.
  * fast: one qrec_svdpp_epoch_usermajor_f32 epoch on synthetic.make_interactions(1M, 100K, 50), d = 64, ratings
    drawn from {0.5, 1, ..., 4}, the GPU filled, users longest first.  Reported with entries/s, the closed form's
    byte model (per entry: Y[i] read twice, Q[i] read, Q[i] / Y[i] deltas and B added: 6 rows + column, rating, Bi;
    per user: P row read and written) against 3.35 TB/s (the H100 SXM's HBM3 data-sheet rate), and the literal
    per-entry form's bytes beside it (every entry reads and writes all W rows of the user).  The tables must stay
    finite."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

U, I, DEG, D = 1_000_000, 100_000, 50, 64
HBM = 3.35e12
REGS = (0.01, 0.01, 0.1, 0.01)                     # SVD++.conf: regU, regI, regB, regY
LR = 0.02


def card(torch):
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        limit = 'unknown (%s)' % e
    return torch.cuda.get_device_name(0), limit


def timed(torch, fn, reps=3):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def parity(torch, E, name, limit):
    from oracle import svdpp_oracle as S
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'svdpp_filmtrust.npz'))
    u, i, (rowptr, cols, _), _, _ = S.golden_ids(g)
    r = g['train_rating']
    gm = float(g['global_mean'])
    init = S.initial_tables(g)
    t0 = time.perf_counter()
    S.svdpp_sgd_sequential(*[t.copy() for t in init], u, i, r, rowptr, cols, LR, *REGS, gm)
    cpu_s = time.perf_counter() - t0
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
    for dt in (torch.float64, torch.float32):
        tabs = [dev(t).to(dt) for t in init]
        args = (dev(u), dev(i), dev(r).to(dt), dev(rowptr), dev(cols))
        loss = torch.zeros(1, dtype=torch.float64, device='cuda')
        run = lambda: E.svdpp_sgd_ordered(*tabs, *args, LR, *REGS, gm, loss)   # noqa: E731
        run()
        ms = timed(torch, run, reps=3)
        print(json.dumps(dict(bench='svdpp_parity_epoch', dtype=str(dt).split('.')[-1], entries=int(len(u)), d=10,
                              ms=round(ms, 3), entries_per_s=len(u) / (ms * 1e-3),
                              numpy_oracle_cpu_ms=round(cpu_s * 1e3, 1), speedup_vs_cpu=cpu_s * 1e3 / ms,
                              card=name, power_limit=limit)), flush=True)


def fast(torch, E, name, limit):
    from qrec_b200.synthetic import make_interactions
    data = make_interactions(U, I, DEG)
    cols = data['i'].contiguous()
    n = int(cols.shape[0])
    rowptr = torch.arange(U + 1, dtype=torch.int64, device='cuda') * DEG
    gen = torch.Generator(device='cuda')
    gen.manual_seed(7)
    vals = torch.randint(1, 9, (n,), device='cuda', generator=gen).float() / 2
    gm = float(vals.double().mean())
    order = torch.from_numpy(E.als_row_order(rowptr.cpu().numpy())).cuda()
    P, Q = torch.rand(U, D, device='cuda', generator=gen) / 3, torch.rand(I, D, device='cuda', generator=gen) / 3
    Y = torch.rand(I, D, device='cuda', generator=gen)
    Bu, Bi = torch.rand(U, device='cuda', generator=gen), torch.rand(I, device='cuda', generator=gen)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    run = lambda: E.svdpp_epoch_usermajor(P, Q, Y, Bu, Bi, rowptr, cols, vals, order, LR, *REGS, gm, loss)  # noqa: E731
    run()
    loss.zero_()
    ms = timed(torch, run, reps=3)
    row = D * 4
    model = n * (6 * row + 12) + U * (2 * row + 16 + 8)
    literal = n * (2 * DEG * row + 2 * row + 12) + U * (2 * row + 16 + 8)
    finite = all(bool(torch.isfinite(t).all()) for t in (P, Q, Y, Bu, Bi))
    print(json.dumps(dict(bench='svdpp_fast_epoch', users=U, items=I, entries=n, d=D, ms=round(ms, 3),
                          entries_per_s=n / (ms * 1e-3), model_bytes=model, model_tb_per_s=model / (ms * 1e-3) / 1e12,
                          share_of_3_35_tb_per_s=model / (ms * 1e-3) / HBM, literal_form_bytes=literal,
                          epoch_rmse=float((loss.item() / 3 / n) ** 0.5), tables_finite=finite,
                          card=name, power_limit=limit)), flush=True)
    assert finite, 'fast epoch left non-finite values in the tables'


def main():
    import torch
    from qrec_b200 import engine as E
    torch.cuda.set_device(0)
    name, limit = card(torch)
    parity(torch, E, name, limit)
    fast(torch, E, name, limit)


if __name__ == '__main__':
    main()
