#!/usr/bin/env python
"""SoRec's trust-edge pass (K9 kind 3), RSTE's rating pass (K16), EE's rating pass (K9 kind 5), the user passes of
SocialMF, SoReg and SREE (K17) and SoReg's pair similarities (qrec_knn_pair_similarity_f64), in float64 as the parity path runs them, on the two synthetic shapes of bench_serec.py (qrec_b200.synthetic, Zipf-skewed item popularity):
  * lastfm-like: 1,892 users x 17,632 items, 40 entries per user, d = 20;
  * yelp2018-like: 31,668 users x 38,048 items, 36 entries per user, d = 64.
Followee counts are bench_serec.py's draw (a fifth of the users follow nobody, the rest a log-normal count); the
followees are drawn uniformly among the other users, weight 1.  The entry stream and the edge list are shuffled.

Timed with CUDA events, one launch per pass: SoRec's edge pass, RSTE's rating pass, and K9 PMF (kind 1) on the same
entry stream, so that the cost of the followee reads shows; EE's rating pass beside K9 SVD (kind 2) on the same entry
stream and bias vectors, so that the cost of the distance form shows; SocialMF's, SoReg's and SREE's user passes over a
shuffled visiting order of all users (followers are the transpose of the followees; SoReg's similarities are drawn uniformly); and the
Pearson similarity of every trust edge over the users' rated rows (half-step ratings), built once per model.  The host wait numbers are prepared beforehand.  The passes
are launched through the C entry points: the engine wrappers' input checks read device values back (ids, CSR bounds),
which would put host round trips inside the timed window of some passes and not others.  Each pass zeroes its row
counters and ticket inside the window (two memsets), as every ordered launch needs.  One JSON line per shape with the
milliseconds per pass, each pass's dependency-chain depth, entries per second, and the card's name and power limit."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_expomf import card, timed   # noqa: E402
from bench_serec import degrees        # noqa: E402

SHAPES = (('lastfm', 1892, 17632, 40, 20, 3), ('yelp2018', 31668, 38048, 36, 64, 2))   # name, U, I, per user, d, reps


def followees(U, seed=3):
    rng = np.random.default_rng(seed)
    deg = degrees(U)
    rowptr = np.zeros(U + 1, np.int64)
    rowptr[1:] = np.cumsum(deg)
    cols = np.empty(rowptr[-1], np.int32)
    for a in range(U):
        pick = rng.choice(U - 1, size=int(deg[a]), replace=False)
        cols[rowptr[a]:rowptr[a + 1]] = pick + (pick >= a)             # anyone but a
    return rowptr, cols


def main():
    import torch
    from qrec_b200 import engine as E, synthetic
    assert torch.cuda.is_available(), 'bench_social_rating needs a GPU'
    torch.cuda.set_device(0)
    name, limit = card(torch)
    f64, dev = torch.float64, torch.device('cuda')
    for label, U, I, per_user, D, reps in SHAPES:
        data = synthetic.make_interactions(U, I, per_user, zipf=True)
        rng = np.random.default_rng(1)
        perm = rng.permutation(data['u'].shape[0])
        u = data['u'].cpu().numpy().astype(np.int32)[perm]
        i = data['i'].cpu().numpy().astype(np.int32)[perm]
        n = u.shape[0]
        r = torch.from_numpy(rng.integers(1, 9, n) * 0.5).to(dev, f64)
        rowptr, cols = followees(U)
        w = np.ones(cols.shape[0])
        denom = np.diff(rowptr).astype(np.float64)
        social = (torch.from_numpy(rowptr).to(dev), torch.from_numpy(cols).to(dev), torch.from_numpy(w).to(dev),
                  torch.from_numpy(denom).to(dev))
        eu = np.repeat(np.arange(U, dtype=np.int32), np.diff(rowptr))
        eperm = rng.permutation(eu.shape[0])
        eu, ev = eu[eperm], cols[eperm]
        g = torch.Generator(device='cuda').manual_seed(1)
        P = torch.rand(U, D, device=dev, dtype=f64, generator=g) / 3
        Q = torch.rand(I, D, device=dev, dtype=f64, generator=g) / 3
        Z = torch.rand(U, D, device=dev, dtype=f64, generator=g) / 10
        loss = torch.zeros(1, dtype=f64, device=dev)
        du, di = torch.from_numpy(u).to(dev), torch.from_numpy(i).to(dev)

        wu, wi, wr, pr, pos, rste_depth = E.rste_order_prepare(u, i, U, I, rowptr, cols)
        rste_dev = [torch.from_numpy(a).to(dev) for a in (wu, wi, wr, pr, pos)]
        mwu, mwi = (torch.from_numpy(a).to(dev) for a in E.mf_order_prepare(u, i, U, I))
        pmf_depth = E.mf_order_depth(u, i, U, I)
        ewu, ewv = (torch.from_numpy(a).to(dev) for a in E.mf_order_prepare(eu, ev, U, U))
        edge_depth = E.mf_order_depth(eu, ev, U, U)
        due, dve = torch.from_numpy(eu).to(dev), torch.from_numpy(ev).to(dev)
        te = torch.rand(eu.shape[0], device=dev, dtype=f64, generator=g)

        def width(m, depth):
            return int(min(2368, max(64, 16 * m / max(1, depth))))

        # raw launches (see the docstring); counters: ver_p | ver_q (or ver_z) | reads_p, and one ticket per pass
        ptr = lambda t: t.data_ptr()                                    # noqa: E731
        st = torch.cuda.current_stream().cuda_stream
        rste_n, pmf_n, edge_n = width(n, rste_depth), width(n, pmf_depth), width(eu.shape[0], edge_depth)
        rste_cnt, pmf_cnt, edge_cnt = (torch.zeros(c, dtype=torch.int32, device=dev) for c in (2 * U + I, U + I, 2 * U))
        tickets = torch.zeros(3, dtype=torch.int64, device=dev)

        def rste():
            rste_cnt.zero_(); tickets[0:1].zero_()
            E.check(E.lib.qrec_rste_sgd_ordered_f64(
                ptr(P), ptr(Q), D, n, ptr(du), ptr(di), ptr(r), *(ptr(a) for a in rste_dev), *(ptr(a) for a in social),
                ptr(rste_cnt), ptr(rste_cnt) + 4 * U, ptr(rste_cnt) + 4 * (U + I), ptr(tickets), 1e-3, 1e-3, 1e-3, 0.6,
                ptr(loss), rste_n, st), 'qrec_rste_sgd_ordered_f64')

        def pmf():
            pmf_cnt.zero_(); tickets[1:2].zero_()
            E.check(E.lib.qrec_mf_sgd_ordered_f64(
                1, ptr(P), ptr(Q), D, n, ptr(du), ptr(di), ptr(r), ptr(mwu), ptr(mwi), ptr(pmf_cnt),
                ptr(pmf_cnt) + 4 * U, ptr(tickets) + 8, 1e-3, 1e-3, 1e-3, None, None, 0.0, 0.0, ptr(loss), pmf_n, st),
                'qrec_mf_sgd_ordered_f64')

        Bu = torch.rand(U, device=dev, dtype=f64, generator=g) / 10
        Bi = torch.rand(I, device=dev, dtype=f64, generator=g) / 10
        btickets = torch.zeros(2, dtype=torch.int64, device=dev)

        def biased(kind, slot):                                         # K9 kind 2 (SVD) or kind 5 (EE)
            def run():
                pmf_cnt.zero_(); btickets[slot:slot + 1].zero_()
                E.check(E.lib.qrec_mf_sgd_ordered_f64(
                    kind, ptr(P), ptr(Q), D, n, ptr(du), ptr(di), ptr(r), ptr(mwu), ptr(mwi), ptr(pmf_cnt),
                    ptr(pmf_cnt) + 4 * U, ptr(btickets) + 8 * slot, 1e-3, 1e-3, 1e-3, ptr(Bu), ptr(Bi), 1e-3, 3.0,
                    ptr(loss), pmf_n, st), 'qrec_mf_sgd_ordered_f64')
            return run

        def edges():
            edge_cnt.zero_(); tickets[2:3].zero_()
            E.check(E.lib.qrec_mf_sgd_ordered_f64(
                E.SOREC_EDGES, ptr(P), ptr(Z), D, eu.shape[0], ptr(due), ptr(dve), ptr(te), ptr(ewu), ptr(ewv),
                ptr(edge_cnt), ptr(edge_cnt) + 4 * U, ptr(tickets) + 16, 1e-3, 0.1, 0.1, None, None, 0.0, 0.0,
                ptr(loss), edge_n, st), 'qrec_mf_sgd_ordered_f64')

        # K17: the user passes over a shuffled visiting order; followers = the followees' transpose
        gorder = np.argsort(cols, kind='stable')
        grp = np.zeros(U + 1, np.int64)
        grp[1:] = np.cumsum(np.bincount(cols, minlength=U))
        gcols = np.repeat(np.arange(U, dtype=np.int32), np.diff(rowptr))[gorder]
        visit = rng.permutation(U).astype(np.int32)
        spos, social_depth = E.social_order_prepare(visit, U, rowptr, cols, grp, gcols)
        sdev = [torch.from_numpy(a).to(dev) for a in (visit, spos, grp, gcols)]
        sim_f = torch.rand(cols.shape[0], device=dev, dtype=f64, generator=g)
        sim_g = torch.rand(cols.shape[0], device=dev, dtype=f64, generator=g)
        social_n = width(U, social_depth)
        done = torch.zeros(U, dtype=torch.int32, device=dev)
        stickets = torch.zeros(3, dtype=torch.int64, device=dev)

        def user_pass(kind):
            def run():
                done.zero_(); stickets[kind:kind + 1].zero_()
                E.check(E.lib.qrec_social_user_pass_f64(
                    kind, ptr(P), D, U, ptr(sdev[0]), ptr(sdev[1]), ptr(social[0]), ptr(social[1]),
                    ptr(social[2]) if kind == 0 else ptr(sim_f), ptr(sdev[2]), ptr(sdev[3]), ptr(sim_g), ptr(done),
                    ptr(stickets) + 8 * kind, 1e-3, 0.1, ptr(loss), social_n, st), 'qrec_social_user_pass_f64')
            return run

        def sree():
            done.zero_(); stickets[2:3].zero_()
            E.check(E.lib.qrec_sree_user_pass_f64(
                ptr(P), D, U, ptr(sdev[0]), ptr(sdev[1]), ptr(social[0]), ptr(social[1]), ptr(social[2]), ptr(sdev[2]),
                ptr(sdev[3]), ptr(done), ptr(stickets) + 16, 1e-3, 0.5, ptr(loss), social_n, st),
                'qrec_sree_user_pass_f64')

        # SoReg's similarities: one per trust edge, over each user's distinct rated items
        up = np.unique(np.stack([u, i]), axis=1)
        krp = np.concatenate([[0], np.bincount(up[0], minlength=U).cumsum()]).astype(np.int64)
        kv = rng.integers(1, 9, up.shape[1]) * 0.5
        km = np.bincount(up[0], weights=kv, minlength=U) / np.maximum(np.diff(krp), 1)
        kdev = [torch.from_numpy(a).to(dev) for a in (krp, up[1].astype(np.int32), kv, E.knn_squares(krp, kv, km, 0), km)]
        ksorted = E.knn_sorted_view(kdev[0], kdev[1], kdev[2]) + E.knn_sorted_view(kdev[0], kdev[1], kdev[3])[1:]
        pa, pb = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (eu, ev))
        pw = torch.ones(eu.shape[0], dtype=f64, device=dev)
        sims = torch.empty(eu.shape[0], dtype=f64, device=dev)

        def pair_sims():
            E.check(E.lib.qrec_knn_pair_similarity_f64(*(ptr(a) for a in kdev), *(ptr(a) for a in ksorted),
                                                       eu.shape[0], ptr(pa), ptr(pb), ptr(pw), ptr(sims), st),
                    'qrec_knn_pair_similarity_f64')

        socialmf, soreg = user_pass(0), user_pass(1)
        svd, ee = biased(2, 0), biased(E.EE_RATINGS, 1)
        for fn in (rste, pmf, edges, socialmf, soreg, pair_sims, svd, ee, sree):      # warm-up
            fn()
        t_rste, t_pmf, t_edges = timed(torch, rste, reps), timed(torch, pmf, reps), timed(torch, edges, reps)
        t_socialmf, t_soreg, t_sims = timed(torch, socialmf, reps), timed(torch, soreg, reps), timed(torch, pair_sims, reps)
        t_svd, t_ee, t_sree = timed(torch, svd, reps), timed(torch, ee, reps), timed(torch, sree, reps)
        print(json.dumps(dict(
            shape=label, users=U, items=I, entries=n, d=D, dtype='float64', edges=int(eu.shape[0]),
            followee_reads=int(np.diff(rowptr)[u].sum()), deg_mean=round(float(np.diff(rowptr).mean()), 2),
            deg_max=int(np.diff(rowptr).max()),
            ms_sorec_edge_pass=round(t_edges, 3), ms_rste_pass=round(t_rste, 3), ms_pmf_pass=round(t_pmf, 3),
            ms_socialmf_user_pass=round(t_socialmf, 3), ms_soreg_user_pass=round(t_soreg, 3),
            ms_soreg_pair_similarity=round(t_sims, 3),
            depth_sorec_edges=edge_depth, depth_rste=rste_depth, depth_pmf=pmf_depth, depth_social_users=social_depth,
            entries_per_s_sorec_edges=round(eu.shape[0] / (t_edges / 1e3)), entries_per_s_rste=round(n / (t_rste / 1e3)),
            entries_per_s_pmf=round(n / (t_pmf / 1e3)),
            ms_svd_pass=round(t_svd, 3), ms_ee_pass=round(t_ee, 3), ms_sree_user_pass=round(t_sree, 3),
            entries_per_s_svd=round(n / (t_svd / 1e3)), entries_per_s_ee=round(n / (t_ee / 1e3)),
            gpu=name, power_limit=limit)), flush=True)


if __name__ == '__main__':
    main()
