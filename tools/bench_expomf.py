#!/usr/bin/env python
"""K13 (ExpoMF) on synthetic sets of the size of two public ranking data sets (qrec_b200.synthetic, Zipf-skewed item
popularity, every user with the same number of distinct items):
  * lastfm as ExpoMF.conf splits it: 1,889 users x 15,423 items, 40 items per user, d = 50;
  * yelp2018: 31,668 users x 38,048 items, 36 items per user, d = 64.

Timed with CUDA events, after a warm-up epoch: the user half (qrec_expomf_solve_rows_f32 against beta), the item half
with the fused exposure prior, and the whole epoch.  One JSON line per shape with the milliseconds, the float64 FMAs
counted from the shapes, the resulting FLOP/s (2 per FMA) and the card's name and power limit.  Per half, every
(row, column) pair costs the tiled accumulation of its weighted outer product, tiles(d) * 16 FMAs with
tiles(d) = ceil(d/4) * (ceil(d/4) + 1) / 2, plus a d-long dot for its posterior; the item half adds one more d-long
dot per pair for the prior.  The observed entries' correction pass is left out of the count (under 0.3 % here)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = (('lastfm', 1889, 15423, 40, 50, 5), ('yelp2018', 31668, 38048, 36, 64, 2))   # name, U, I, per user, d, reps
LAM, LAM_Y = 1e-5, 1.0


def card(torch):
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        limit = 'unknown (%s)' % e
    return torch.cuda.get_device_name(0), limit


def timed(torch, fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def fmas(U, I, d):
    """float64 FMAs of one user half and of one item half with the prior."""
    nb = (d + 3) // 4
    pairs = U * I
    half = pairs * (nb * (nb + 1) // 2) * 16 + pairs * d
    return half, half + pairs * d


def main():
    import torch
    from qrec_b200 import engine as E, synthetic
    assert torch.cuda.is_available(), 'bench_expomf needs a GPU'
    torch.cuda.set_device(0)
    name, limit = card(torch)
    for label, U, I, deg, D, reps in SHAPES:
        data = synthetic.make_interactions(U, I, deg, zipf=True)
        u, i = data['u'], data['i']
        n = u.shape[0]
        urp, ucol = data['sorted_rowptr'], data['sorted_cols']
        order = torch.argsort(i, stable=True)
        irp = torch.zeros(I + 1, dtype=torch.int64, device='cuda')
        torch.cumsum(torch.bincount(i, minlength=I), 0, out=irp[1:])
        icol = u[order].contiguous()
        uord = torch.from_numpy(E.als_row_order(urp.cpu().numpy())).cuda()
        iord = torch.from_numpy(E.als_row_order(irp.cpu().numpy())).cuda()
        g = torch.Generator(device='cuda').manual_seed(1)
        theta = torch.randn(U, D, device='cuda', generator=g) * 0.01
        beta = torch.randn(I, D, device='cuda', generator=g) * 0.01
        mu = torch.full((I,), 0.01, device='cuda')
        nxt = torch.empty_like(mu)
        n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')

        def user_half():
            E.expomf_half_epoch(theta, beta, urp, ucol, mu, False, LAM, LAM_Y, uord, n_failed=n_failed)

        def item_half():
            E.expomf_half_epoch(beta, theta, irp, icol, mu, True, LAM, LAM_Y, iord, mu_out=nxt, n_failed=n_failed)

        def epoch():
            nonlocal mu, nxt
            user_half()
            item_half()
            mu, nxt = nxt, mu

        epoch()                                                         # warm-up
        t_user = timed(torch, user_half, reps)
        t_item = timed(torch, item_half, reps)
        t_epoch = timed(torch, epoch, reps)
        f_user, f_item = fmas(U, I, D)
        print(json.dumps(dict(
            bench='expomf', shape=label, users=U, items=I, interactions=n, d=D, reps=reps,
            user_half_ms=round(t_user, 3), item_half_with_prior_ms=round(t_item, 3), epoch_ms=round(t_epoch, 3),
            user_half_fma64=f_user, item_half_fma64=f_item,
            user_half_tflops=round(2 * f_user / t_user / 1e9, 3), item_half_tflops=round(2 * f_item / t_item / 1e9, 3),
            epoch_tflops=round(2 * (f_user + f_item) / t_epoch / 1e9, 3),
            failed_systems=int(n_failed.item()), gpu=name, power_limit=limit)), flush=True)


if __name__ == '__main__':
    main()
