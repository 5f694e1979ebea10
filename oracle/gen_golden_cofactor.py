#!/usr/bin/env python
"""Golden run of the reference's CoFactor (model/ranking/CoFactor.py with base/iterativeRecommender.py around it),
UNMODIFIED, through its QRec driver on FilmTrust.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose
work-directory setup it shares: the GPU box never runs it.

Recorded in tests/golden/cofactor_filmtrust.npz:
  * the training / test lists as the model holds them and the id maps (user_names / item_names);
  * the SPPMI matrix of initModel as a CSR over item ids with ascending columns (float64);
  * X, Y, w, c after the last epoch, G's rows after the last epoch for the items that have SPPMI contexts (the
    others keep their initial draw), and every ROW_STRIDE-th row of Y and G after every epoch.  The initial state
    is not stored: X0 = 10 P, Y0 = 10 Q, w0, c0, G0 come from the seeded legacy numpy stream, which the generator
    checks (oracle/cofactor_oracle.py: initial_state);
  * the epoch losses (captured from the reference's `epoch:` line: CoFactor has no isConverged) and the final
    measure lines.

Usage:  python oracle/gen_golden_cofactor.py   (writes tests/golden/cofactor_filmtrust.npz)
"""
import contextlib
import io
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen_golden import OUT, _enter_workdir   # noqa: E402
from oracle import cofactor_oracle as CO     # noqa: E402

CONF_COFACTOR = """ratings=./dataset/FilmTrust/trainset.txt
ratings.setup=-columns 0 1 2
model.name=CoFactor
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt
item.ranking=on -topN 10
num.factors=20
num.max.epoch=3
learnRate=-init 0.05 -max 1
reg.lambda=-u 1 -i 0.01 -b 0.01 -s 0.1
CoFactor=-k 5 -gamma 0.01 -filter 2
output.setup=on -dir ./results/
"""
SEED = 23
ROW_STRIDE = 16    # rows kept of Y and G after every epoch (keeps the fixture under 1 MB)


def gen_cofactor():
    from util.config import ModelConf
    from QRec import QRec
    import model.ranking.CoFactor as M
    with open('CoFactor_ft.conf', 'w') as f:
        f.write(CONF_COFACTOR)
    random.seed(SEED)
    np.random.seed(SEED)
    conf = ModelConf('CoFactor_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    model = M.CoFactor(conf, q.trainingData, q.testData)
    train, test = list(model.data.trainingData), list(model.data.testData)
    rec = dict(X=[], Y=[], G=[], w=[], c=[], loss=[])

    def spy_print(*args, **kw):
        # trainModel's per-epoch line `epoch: e loss: l` (CoFactor.py, end of the epoch loop)
        if args and args[0] == 'epoch:':
            for k in ('X', 'Y', 'G', 'w', 'c'):
                rec[k].append(getattr(model, k).copy())
            rec['loss'].append(float(model.loss))
        print(*args, **kw)

    M.print = spy_print
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            model.readConfiguration()
            model.initializing_log()
            model.initModel()
            P0, Q0 = model.P.copy(), model.Q.copy()
            model.trainModel()
            model.evalRanking()
    finally:
        del M.print
    measure = [m.strip() for m in model.measure]
    ids = model.data.item
    n_items = len(ids)
    rows = [dict() for _ in range(n_items)]
    for a, row in model.SPPMI.items():
        for b, v in row.items():
            rows[ids[a]][ids[b]] = v
    rowptr = np.zeros(n_items + 1, dtype=np.int64)
    cols, vals = [], []
    for k, row in enumerate(rows):
        for b in sorted(row):
            cols.append(b)
            vals.append(row[b])
        rowptr[k + 1] = len(cols)
    has_ctx = np.diff(rowptr) > 0
    g = dict(seed=np.array(SEED), user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
             item_names=np.array([model.data.id2item[k] for k in range(n_items)]))
    X0, Y0, w0, c0, G0 = CO.initial_state(g, model.emb_size)
    assert np.array_equal(P0 * 10, X0) and np.array_equal(Q0 * 10, Y0)
    G_last = rec['G'][-1]
    assert np.array_equal(G_last[~has_ctx], G0[~has_ctx])
    assert np.array_equal(rec['w'][-1][~has_ctx], w0[~has_ctx]) and np.array_equal(rec['c'][-1][~has_ctx], c0[~has_ctx])
    print('CoFactor FilmTrust: train', model.data.trainingSize(), 'SPPMI nnz', len(cols), 'items with contexts',
          int(has_ctx.sum()), 'losses', rec['loss'], 'measure', measure)
    np.savez_compressed(
        os.path.join(OUT, 'cofactor_filmtrust.npz'),
        train_users=np.array([e[0] for e in train]), train_items=np.array([e[1] for e in train]),
        train_rating=np.array([e[2] for e in train], dtype=np.float64),
        test_users=np.array([e[0] for e in test]), test_items=np.array([e[1] for e in test]),
        test_rating=np.array([e[2] for e in test], dtype=np.float64),
        sppmi_rowptr=rowptr, sppmi_cols=np.array(cols, dtype=np.int32), sppmi_vals=np.array(vals),
        X_last=rec['X'][-1], Y_last=rec['Y'][-1], w_last=rec['w'][-1], c_last=rec['c'][-1],
        G_last_ctx=G_last[has_ctx], row_stride=np.array(ROW_STRIDE),
        Y_rows_epoch=np.stack([y[::ROW_STRIDE] for y in rec['Y']]),     # [E, ceil(I / ROW_STRIDE), d] float64
        G_rows_epoch=np.stack([x[::ROW_STRIDE] for x in rec['G']]),
        loss=np.array(rec['loss']), measure=np.array(measure), conf=np.array(CONF_COFACTOR), **g)


if __name__ == '__main__':
    _enter_workdir()
    gen_cofactor()
