#!/usr/bin/env python
"""K15 (UserKNN, ItemKNN, SlopeOne) on synthetic sets of the size of two public data sets (qrec_b200.synthetic,
Zipf-skewed item popularity, every user with the same number of distinct items), ratings drawn in half steps from a
seeded stream, and a held-out test list of one line for each of a seeded fifth of the users:
  * lastfm: 1,892 users x 17,632 items, 40 items per user;
  * yelp2018: 31,668 users x 38,048 items, 36 items per user.

Timed with CUDA events after a warm-up, pcc with 20 neighbours: the neighbour build (engine.knn_neighbours) and the
prediction of every test line (engine.knn_predict) of each KNN model, and SlopeOne's fused launch
(engine.slopeone_predict).  The host work around them (squares, transposes, checks) is not timed.  One JSON line per
shape with the milliseconds, the co-rated terms the scatter visits (counted from the shapes on the host: for every
query entry, the length of its column on the other side), terms per second, and the card's name and power limit."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_expomf import card, timed   # noqa: E402

SHAPES = (('lastfm', 1892, 17632, 40, 3), ('yelp2018', 31668, 38048, 36, 2))   # name, U, I, per user, reps
K = 20


def side(rowptr, cols, vals, n_cols):
    """The other side's CSR of the same entries, each row in the order of the first side's rows."""
    rows = np.repeat(np.arange(len(rowptr) - 1, dtype=np.int32), np.diff(rowptr))
    order = np.argsort(cols, kind='stable')
    rp = np.zeros(n_cols + 1, dtype=np.int64)
    rp[1:] = np.cumsum(np.bincount(cols, minlength=n_cols))
    return rp, rows[order], vals[order]


def main():
    import torch
    from qrec_b200 import engine as E, synthetic
    assert torch.cuda.is_available(), 'bench_knn needs a GPU'
    name_card, limit = card(torch)
    for name, U, I, deg, reps in SHAPES:
        data = synthetic.make_interactions(U, I, deg, zipf=True)
        ucols = data['i'].cpu().numpy().astype(np.int32)
        rng = np.random.default_rng(11)
        uvals = rng.integers(1, 11, ucols.shape[0]).astype(np.float64) / 2
        urp = np.arange(U + 1, dtype=np.int64) * deg
        irp, icols, ivals = side(urp, ucols, uvals, I)
        test_users = np.sort(rng.choice(U, U // 5, replace=False)).astype(np.int32)
        test_items = ucols[urp[test_users] + rng.integers(0, deg, test_users.shape[0])].astype(np.int32)
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
        means_u = np.add.reduceat(uvals, urp[:-1]) / deg
        means_i = np.array([ivals[irp[k]:irp[k + 1]].sum() / max(irp[k + 1] - irp[k], 1) for k in range(I)])
        line = dict(shape=name, users=U, items=I, ratings=int(ucols.shape[0]), test_lines=int(test_users.shape[0]),
                    K=K, similarity='pcc', card=name_card, power_limit=limit)
        for model, rp, cl, vl, means, qrows, probes, ncols, other_rp in (
                ('UserKNN', urp, ucols, uvals, means_u, test_users, test_items, I, irp),
                ('ItemKNN', irp, icols, ivals, means_i, None, test_users, U, urp)):
            if qrows is None:       # the test items in order of first appearance, and each line's position
                uniq, first = np.unique(test_items, return_index=True)
                qrows = uniq[np.argsort(first)].astype(np.int32)
            qpos_of = {int(r): p for p, r in enumerate(qrows)}
            lq = np.array([qpos_of[int(r)] for r in (test_users if model == 'UserKNN' else test_items)], np.int32)
            sq = E.knn_squares(rp, vl, means, 0)
            d = [cu(a) for a in (rp, cl, vl, sq, means, qrows)]
            run_nb = lambda: E.knn_neighbours(d[0], d[1], d[2], d[3], d[4], ncols, d[5], 0, K)   # noqa: E731
            out = run_nb()
            ms_nb = timed(torch, run_nb, reps)
            lq_d, lp_d = cu(lq), cu(probes.astype(np.int32))
            sv = E.knn_sorted_view(d[0], d[1], d[2])
            run_pr = lambda: E.knn_predict(d[0], *sv, d[4], 3.0, d[5], *out, lq_d, lp_d, model == 'UserKNN')  # noqa: E731
            run_pr()
            ms_pr = timed(torch, run_pr, reps)
            col_len = np.diff(other_rp)
            terms = int(sum(col_len[cl[rp[q]:rp[q + 1]]].sum() for q in qrows.tolist()))
            line[model] = dict(neighbours_ms=round(ms_nb, 3), predict_ms=round(ms_pr, 3), queries=int(qrows.shape[0]),
                               corated_terms=terms, terms_per_s=terms / (ms_nb * 1e-3))
        uniq, first = np.unique(test_items, return_index=True)
        titems = uniq[np.argsort(first)].astype(np.int32)
        pos = {int(r): p for p, r in enumerate(titems)}
        lq = cu(np.array([pos[int(i)] for i in test_items], np.int32))
        s = [cu(a) for a in (irp, icols, ivals, means_i, urp, ucols, uvals, means_u, titems)]
        lu = cu(test_users)
        run_so = lambda: E.slopeone_predict(*s[:8], 3.0, s[8], lq, lu)   # noqa: E731
        run_so()
        ms_so = timed(torch, run_so, reps)
        col_len = np.diff(urp)
        terms = int(sum(col_len[icols[irp[q]:irp[q + 1]]].sum() for q in titems.tolist()))
        line['SlopeOne'] = dict(ms=round(ms_so, 3), test_items=int(titems.shape[0]), corated_terms=terms,
                                terms_per_s=terms / (ms_so * 1e-3))
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
