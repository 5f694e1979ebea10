#!/usr/bin/env python
"""K12 (CoFactor) on a synthetic set of the size of a public ranking data set (yelp2018: 31K users, 38K items, 1.2M
interactions): 100K users x 40K items x 20 items per user with Zipf-skewed popularity (qrec_b200.synthetic),
ratings 1, d = 64, the CoFactor.conf values (-k 5 -gamma 0.01 -filter 2, regU 1).

Timed with CUDA events, after a warm-up: the SPPMI build (engine.sppmi_csr: co-occurrence counts, PMI, compaction,
normalisation), the user half-epoch (Gram of Y + qrec_als_solve_rows_*) and the item half-epoch (Gram of X +
qrec_cofactor_item_sweep_*), on float64 and on float32 tables.  One JSON line per table type, with the SPPMI's
nnz, the number of items with contexts, the Gauss-Seidel dependency depth of the in-order item sweep (the longest
chain of items that must run one after another), and the card's name and power limit."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

U, I, DEG, D = 100_000, 40_000, 20, 64
K, GAMMA, FILTER, REG, ALPHA = 5, 0.01, 2, 1.0, 10.0


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


def main():
    import numpy as np
    import torch
    from qrec_b200 import engine as E, synthetic
    from oracle.cofactor_oracle import gauss_seidel_depth
    assert torch.cuda.is_available(), 'bench_cofactor needs a GPU'
    torch.cuda.set_device(0)
    name, limit = card(torch)
    data = synthetic.make_interactions(U, I, DEG, zipf=True)
    u, i = data['u'], data['i']
    n = u.shape[0]
    urp = data['sorted_rowptr']
    ucol = data['sorted_cols']
    order = torch.argsort(i, stable=True)
    irp = torch.zeros(I + 1, dtype=torch.int64, device='cuda')
    torch.cumsum(torch.bincount(i, minlength=I), 0, out=irp[1:])
    icol = u[order].contiguous()
    uord = torch.from_numpy(E.als_row_order(urp.cpu().numpy())).cuda()
    E.sppmi_csr(irp, icol, U, K, FILTER)                               # warm-up
    t_sppmi = timed(torch, lambda: E.sppmi_csr(irp, icol, U, K, FILTER))
    srp, scol, sval = E.sppmi_csr(irp, icol, U, K, FILTER)
    srp_h, scol_h = srp.cpu().numpy(), scol.cpu().numpy()
    depth = gauss_seidel_depth(srp_h, scol_h)
    with_ctx = int((np.diff(srp_h) > 0).sum())
    for dt in (torch.float64, torch.float32):
        g = torch.Generator(device='cuda').manual_seed(1)
        X = torch.rand(U, D, device='cuda', dtype=dt, generator=g) * (10 / 3)
        Y = torch.rand(I, D, device='cuda', dtype=dt, generator=g) * (10 / 3)
        G = torch.rand(I, D, device='cuda', dtype=dt, generator=g) / 10
        w = torch.rand(I, device='cuda', dtype=dt, generator=g) / 10
        c = torch.rand(I, device='cuda', dtype=dt, generator=g) / 10
        ones = torch.ones(n, device='cuda', dtype=dt)
        item_csr, sppmi = (irp, icol, ones), (srp, scol, sval.to(dt))
        gram = torch.empty(D, D, dtype=torch.float64, device='cuda')
        ws = torch.empty(int(E.lib.qrec_als_gram_workspace_bytes(U, D)), dtype=torch.uint8, device='cuda')
        loss = torch.zeros(1, dtype=torch.float64, device='cuda')
        n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')

        def user_half():
            E.als_gram(Y, gram, ws)
            E.als_solve_rows(X, Y, gram, urp, ucol, ones, REG, ALPHA, uord, loss=loss, n_failed=n_failed)

        def item_half():
            E.als_gram(X, gram, ws)
            E.cofactor_item_sweep(Y, G, w, c, X, gram, item_csr, sppmi, REG, GAMMA, ALPHA, n_failed=n_failed)

        user_half(); item_half()                                        # warm-up epoch
        t_user = timed(torch, user_half)
        t_item = timed(torch, item_half)
        print(json.dumps(dict(
            bench='cofactor', dtype=str(dt).replace('torch.', ''), users=U, items=I, interactions=n, d=D,
            k=K, gamma=GAMMA, filter=FILTER, sppmi_nnz=int(scol_h.shape[0]), items_with_contexts=with_ctx,
            gauss_seidel_depth=depth, sppmi_ms=round(t_sppmi, 3), user_half_epoch_ms=round(t_user, 3),
            item_half_epoch_ms=round(t_item, 3), epoch_ms=round(t_user + t_item, 3),
            failed_systems=int(n_failed.item()), gpu=name, power_limit=limit)), flush=True)


if __name__ == '__main__':
    main()
