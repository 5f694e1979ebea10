#!/usr/bin/env python
"""K14 (SERec) on synthetic sets of the size of two public ranking data sets (qrec_b200.synthetic, Zipf-skewed item
popularity, every user with the same number of distinct items) with a synthetic trust network:
  * lastfm as SERec.conf reads it: 1,892 users x 17,632 items, 40 items per user, d = 20;
  * yelp2018: 31,668 users x 38,048 items, 36 items per user, d = 64 (the shape of bench_expomf.py).
Followee counts are drawn like lastfm's trust network: a fifth of the users follow nobody, the rest a log-normal
count with a long tail, about 13 per user on average (reported as deg_mean / deg_max).

Timed with CUDA events, after a warm-up epoch: the user half (qrec_serec_solve_rows_f32 against beta with the social
prior), the item half with the fused summed posteriors, and the whole epoch; then ExpoMF's epoch
(qrec_expomf_solve_rows_f32, both halves) on the same tables, so that the cost of the per-pair social prior shows
directly.  One JSON line per shape with the milliseconds, the float64 FMAs counted from the shapes (as in
bench_expomf.py: the tiled accumulation and the posterior's dot per pair, one more dot per pair in the item half; the
prior's few operations per pair are not counted), the resulting FLOP/s and the card's name and power limit."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_expomf import card, fmas, timed   # noqa: E402

SHAPES = (('lastfm', 1892, 17632, 40, 20, 5), ('yelp2018', 31668, 38048, 36, 64, 2))   # name, U, I, per user, d, reps
LAM, LAM_Y = 1e-5 / 0.01, 0.01


def degrees(U, seed=7):
    rng = np.random.default_rng(seed)
    deg = np.rint(rng.lognormal(2.43, 0.85, U)).astype(np.int64)
    deg[rng.random(U) < 0.2] = 0
    return np.minimum(deg, U - 1).astype(np.int32)


def main():
    import torch
    from qrec_b200 import engine as E, synthetic
    assert torch.cuda.is_available(), 'bench_serec needs a GPU'
    torch.cuda.set_device(0)
    name, limit = card(torch)
    for label, U, I, per_user, D, reps in SHAPES:
        data = synthetic.make_interactions(U, I, per_user, zipf=True)
        u, i = data['u'], data['i']
        n = u.shape[0]
        urp, ucol = data['sorted_rowptr'], data['sorted_cols']
        order = torch.argsort(i, stable=True)
        irp = torch.zeros(I + 1, dtype=torch.int64, device='cuda')
        torch.cumsum(torch.bincount(i, minlength=I), 0, out=irp[1:])
        icol = u[order].contiguous()
        uord = torch.from_numpy(E.als_row_order(urp.cpu().numpy())).cuda()
        iord = torch.from_numpy(E.als_row_order(irp.cpu().numpy())).cuda()
        deg_h = degrees(U)
        deg = torch.from_numpy(deg_h).cuda()
        g = torch.Generator(device='cuda').manual_seed(1)
        theta = torch.randn(U, D, device='cuda', generator=g) * 0.5
        beta = torch.randn(I, D, device='cuda', generator=g) * 0.5
        n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
        bufs = [None, torch.empty(I, dtype=torch.float64, device='cuda')]

        def user_half():
            E.serec_half_epoch(theta, beta, urp, ucol, bufs[0], deg, True, LAM, LAM_Y, uord, n_failed=n_failed)

        def item_half():
            E.serec_half_epoch(beta, theta, irp, icol, bufs[0], deg, False, LAM, LAM_Y, iord, asum_out=bufs[1],
                               n_failed=n_failed)

        def epoch():
            user_half()
            item_half()
            bufs[0], bufs[1] = bufs[1], (torch.empty_like(bufs[1]) if bufs[0] is None else bufs[0])

        epoch()                                                         # warm-up; later epochs use the social prior
        t_user = timed(torch, user_half, reps)
        t_item = timed(torch, item_half, reps)
        t_epoch = timed(torch, epoch, reps)
        mu = [torch.full((I,), 0.01, device='cuda'), torch.empty(I, device='cuda')]

        def expomf_epoch():
            E.expomf_half_epoch(theta, beta, urp, ucol, mu[0], False, LAM, LAM_Y, uord, n_failed=n_failed)
            E.expomf_half_epoch(beta, theta, irp, icol, mu[0], True, LAM, LAM_Y, iord, mu_out=mu[1], n_failed=n_failed)
            mu[0], mu[1] = mu[1], mu[0]

        expomf_epoch()
        t_expo = timed(torch, expomf_epoch, reps)
        f_user, f_item = fmas(U, I, D)
        print(json.dumps(dict(
            bench='serec', shape=label, users=U, items=I, interactions=n, d=D, reps=reps,
            deg_mean=round(float(deg_h.mean()), 2), deg_max=int(deg_h.max()), deg_zero=int((deg_h == 0).sum()),
            user_half_ms=round(t_user, 3), item_half_with_asum_ms=round(t_item, 3), epoch_ms=round(t_epoch, 3),
            expomf_epoch_ms=round(t_expo, 3), serec_over_expomf=round(t_epoch / t_expo, 3),
            user_half_fma64=f_user, item_half_fma64=f_item,
            user_half_tflops=round(2 * f_user / t_user / 1e9, 3), item_half_tflops=round(2 * f_item / t_item / 1e9, 3),
            epoch_tflops=round(2 * (f_user + f_item) / t_epoch / 1e9, 3),
            failed_systems=int(n_failed.item()), gpu=name, power_limit=limit)), flush=True)


if __name__ == '__main__':
    main()
