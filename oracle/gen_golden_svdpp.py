#!/usr/bin/env python
"""Golden run of the reference's SVD++ (model/rating/SVDPlusPlus.py with base/iterativeRecommender.py around it),
UNMODIFIED, through its QRec driver on FilmTrust with config/SVD++.conf's values and three epochs.  TEST
INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose work-directory setup it shares: the GPU box never runs it.

Recorded in tests/golden/svdpp_filmtrust.npz:
  * the training / test lists as the model holds them (initial order) and the id maps (user_names / item_names);
  * the order the entries were visited in each epoch (indices into the initial list; isConverged reshuffles);
  * P, Q, Y, Bu, Bi after the last epoch and every ROW_STRIDE-th row of each after every epoch (float64).  The
    initial tables are not stored: they are the seeded legacy numpy draws of initModel, which the generator checks
    (oracle/svdpp_oracle.py: initial_tables);
  * the epoch losses, the learning rate before / after every isConverged, the MT19937 state before initModel and
    after every epoch, the MAE / RMSE lines of every epoch and the final ones.

Usage:  python oracle/gen_golden_svdpp.py   (writes tests/golden/svdpp_filmtrust.npz)
"""
import contextlib
import io
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import OUT, _enter_workdir, _state_to_array   # noqa: E402

CONF_SVDPP = """ratings=./dataset/FilmTrust/trainset.txt
ratings.setup=-columns 0 1 2
model.name=SVDPlusPlus
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt
item.ranking=off -topN 10
num.factors=10
num.max.epoch=3
learnRate=-init 0.02 -max 1
reg.lambda=-u 0.01 -i 0.01 -b 0.1 -s 0.1
SVDPlusPlus=-y 0.01
output.setup=on -dir ./results/
"""
SEED = 11
ROW_STRIDE = 8     # rows kept of the tables after the earlier epochs (keeps the fixture under 1 MB)
TABLES = ('P', 'Q', 'Y', 'Bu', 'Bi')


def gen_svdpp():
    from util.config import ModelConf
    from QRec import QRec
    from model.rating.SVDPlusPlus import SVDPlusPlus
    with open('SVDPP_ft.conf', 'w') as f:
        f.write(CONF_SVDPP)
    random.seed(SEED)
    np.random.seed(SEED)
    conf = ModelConf('SVDPP_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    model = SVDPlusPlus(conf, q.trainingData, q.testData)
    first = list(model.data.trainingData)
    where = {id(e): k for k, e in enumerate(first)}
    rec = dict(order=[], loss=[], lrate=[], states=[], measure=[], **{t: [] for t in TABLES})
    orig_conv = SVDPlusPlus.isConverged

    def spy_conv(self, epoch):
        rec['order'].append(np.array([where[id(e)] for e in self.data.trainingData], dtype=np.uint16))
        for t in TABLES:
            rec[t].append(getattr(self, t).copy())
        rec['loss'].append(float(self.loss))
        lr_before = self.lRate
        r = orig_conv(self, epoch)
        rec['measure'].append([m.strip() for m in self.measure])
        rec['lrate'].append((lr_before, self.lRate))
        rec['states'].append(_state_to_array(random.getstate()))
        return r

    SVDPlusPlus.isConverged = spy_conv
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            model.readConfiguration()
            model.initializing_log()
            state_before = _state_to_array(random.getstate())
            model.initModel()
            init = [getattr(model, t).copy() for t in ('P', 'Q', 'Bu', 'Bi', 'Y')]
            model.trainModel()
            model.evalRatings()
    finally:
        SVDPlusPlus.isConverged = orig_conv
    assert len(first) < 1 << 16
    measure = [m.strip() for m in model.measure]
    r = np.random.RandomState(SEED)
    nu, ni, d = len(model.data.user), len(model.data.item), model.emb_size
    redraw = [r.rand(nu, d) / 3, r.rand(ni, d) / 3, r.rand(nu), r.rand(ni), r.rand(ni, d)]
    assert all(np.array_equal(a, b) for a, b in zip(init, redraw))
    print('SVD++ FilmTrust: train', model.data.trainingSize(), 'losses', rec['loss'], 'measure', measure)
    tables = {}
    for t in TABLES:
        tables[t + '_last'] = rec[t][-1]
        tables[t + '_rows_epoch'] = np.stack([x[::ROW_STRIDE] for x in rec[t]])
    np.savez_compressed(
        os.path.join(OUT, 'svdpp_filmtrust.npz'),
        user_names=np.array([model.data.id2user[k] for k in range(nu)]),
        item_names=np.array([model.data.id2item[k] for k in range(ni)]),
        train_users=np.array([e[0] for e in first]), train_items=np.array([e[1] for e in first]),
        train_rating=np.array([e[2] for e in first], dtype=np.float64),
        test_users=np.array([e[0] for e in model.data.testData]),
        test_items=np.array([e[1] for e in model.data.testData]),
        test_rating=np.array([e[2] for e in model.data.testData], dtype=np.float64),
        global_mean=np.array(model.data.globalMean),
        order_epoch=np.stack(rec['order']),                # [E, n] uint16 indices into the initial list
        row_stride=np.array(ROW_STRIDE), loss=np.array(rec['loss']), lrate=np.array(rec['lrate']),
        mt_state_before=state_before, mt_state_after_epoch=np.stack(rec['states']),
        epoch_measure=np.array(rec['measure']), measure=np.array(measure),
        seed=np.array(SEED), conf=np.array(CONF_SVDPP), **tables)


if __name__ == '__main__':
    _enter_workdir()
    gen_svdpp()
