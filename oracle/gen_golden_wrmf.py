#!/usr/bin/env python
"""Golden run of the reference's WRMF (model/ranking/WRMF.py with base/iterativeRecommender.py around it),
UNMODIFIED, through its QRec driver on FilmTrust.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose
work-directory setup it shares: the GPU box never runs it.

Recorded in tests/golden/wrmf_filmtrust.npz:
  * the training / test lists as the model holds them and the id maps (user_names / item_names);
  * X, Y after the last epoch and every ROW_STRIDE-th row of X, Y after every epoch (float64).  X0, Y0 are not
    stored: they are 10 * the P / Q draws of initModel, np.random.RandomState(seed).rand(...) / 3, which the
    generator checks (oracle/wrmf_oracle.py: initial_tables);
  * the epoch losses, the learning rate before / after every isConverged and the MT19937 state after it
    (isConverged reshuffles trainingData);
  * the final measure lines and the first 64 lines of the top-10 output.

Usage:  python oracle/gen_golden_wrmf.py   (writes tests/golden/wrmf_filmtrust.npz)
"""
import contextlib
import io
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import OUT, _enter_workdir, _state_to_array   # noqa: E402

CONF_WRMF = """ratings=./dataset/FilmTrust/trainset.txt
ratings.setup=-columns 0 1 2
model.name=WRMF
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt
item.ranking=on -topN 10
num.factors=20
num.max.epoch=3
WRMF=-alpha 10 -lamba 1
learnRate=-init 0.01 -max 1
reg.lambda=-u 1 -i 0.02 -b 0.02
output.setup=on -dir ./results/
"""
SEED = 21
ROW_STRIDE = 8     # rows kept of the tables after the earlier epochs (keeps the fixture under 1 MB)


def gen_wrmf():
    from util.config import ModelConf
    from QRec import QRec
    from model.ranking.WRMF import WRMF
    with open('WRMF_ft.conf', 'w') as f:
        f.write(CONF_WRMF)
    random.seed(SEED)
    np.random.seed(SEED)
    conf = ModelConf('WRMF_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    model = WRMF(conf, q.trainingData, q.testData)
    train, test = list(model.data.trainingData), list(model.data.testData)
    rec = dict(X=[], Y=[], loss=[], lrate=[], states=[])
    orig_conv = WRMF.isConverged

    def spy_conv(self, epoch):
        rec['X'].append(self.X.copy())
        rec['Y'].append(self.Y.copy())
        rec['loss'].append(float(self.loss))
        lr_before = self.lRate
        r = orig_conv(self, epoch)
        rec['lrate'].append((lr_before, self.lRate))
        rec['states'].append(_state_to_array(random.getstate()))
        return r

    WRMF.isConverged = spy_conv
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            model.readConfiguration()
            model.initializing_log()
            state_before = _state_to_array(random.getstate())
            model.initModel()
            X0, Y0 = model.X.copy(), model.Y.copy()
            model.trainModel()
            model.evalRanking()
    finally:
        WRMF.isConverged = orig_conv
    measure = [m.strip() for m in model.measure]
    r = np.random.RandomState(SEED)
    P0 = r.rand(len(model.data.user), model.emb_size) / 3
    Q0 = r.rand(len(model.data.item), model.emb_size) / 3
    assert np.array_equal(P0 * 10, X0) and np.array_equal(Q0 * 10, Y0)
    print('WRMF FilmTrust: train', model.data.trainingSize(), 'losses', rec['loss'], 'measure', measure)
    np.savez_compressed(
        os.path.join(OUT, 'wrmf_filmtrust.npz'),
        user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
        item_names=np.array([model.data.id2item[k] for k in range(len(model.data.item))]),
        train_users=np.array([e[0] for e in train]), train_items=np.array([e[1] for e in train]),
        train_rating=np.array([e[2] for e in train], dtype=np.float64),
        test_users=np.array([e[0] for e in test]), test_items=np.array([e[1] for e in test]),
        test_rating=np.array([e[2] for e in test], dtype=np.float64),
        X_last=rec['X'][-1], Y_last=rec['Y'][-1], row_stride=np.array(ROW_STRIDE),
        X_rows_epoch=np.stack([x[::ROW_STRIDE] for x in rec['X']]),     # [E, ceil(n / ROW_STRIDE), d] float64
        Y_rows_epoch=np.stack([y[::ROW_STRIDE] for y in rec['Y']]),
        loss=np.array(rec['loss']), lrate=np.array(rec['lrate']),
        mt_state_before=state_before, mt_state_after_epoch=np.stack(rec['states']),
        measure=np.array(measure), rec_lines=np.array(model.recOutput[1:65]),
        seed=np.array(SEED), conf=np.array(CONF_WRMF))


if __name__ == '__main__':
    _enter_workdir()
    gen_wrmf()
