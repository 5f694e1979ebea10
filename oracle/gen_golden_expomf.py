#!/usr/bin/env python
"""Golden run of the reference's ExpoMF (model/ranking/ExpoMF.py with base/iterativeRecommender.py around it),
UNMODIFIED, through its QRec driver on FilmTrust.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose
work-directory setup it shares: the GPU box never runs it.

The model's `joblib.Parallel` is replaced by a sequential call, so that no worker processes are spawned.  The
batches it hands out are independent (every row reads only the old tables), so the results are the same.

Recorded in tests/golden/expomf_filmtrust.npz:
  * the training / test lists as the model holds them and the id maps (user_names / item_names);
  * theta, beta and mu after every epoch (float32, as the reference keeps them).  The initial state is not stored:
    it comes from the seeded legacy numpy stream (oracle/expomf_oracle.py: initial_state), which the generator checks;
  * the final measure lines.

Usage:  python oracle/gen_golden_expomf.py   (writes tests/golden/expomf_filmtrust.npz)
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
from oracle import expomf_oracle as EO       # noqa: E402

CONF_EXPOMF = """ratings=./dataset/FilmTrust/trainset.txt
ratings.setup=-columns 0 1 2
model.name=ExpoMF
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt
item.ranking=on -topN 10
num.factors=20
num.max.epoch=3
learnRate=-init 0.01 -max 1
reg.lambda=-u 1 -i 0.02 -b 0.02
output.setup=on -dir ./results/
"""
SEED = 5


def sequential_parallel(n_jobs=None, **kw):
    """joblib.Parallel(n_jobs)(delayed(f)(*args) ...) as a plain loop in the calling process."""
    return lambda tasks: [f(*args, **kwargs) for f, args, kwargs in tasks]


def gen_expomf():
    from util.config import ModelConf
    from QRec import QRec
    import model.ranking.ExpoMF as M
    with open('ExpoMF_ft.conf', 'w') as f:
        f.write(CONF_EXPOMF)
    random.seed(SEED)
    np.random.seed(SEED)
    conf = ModelConf('ExpoMF_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    model = M.ExpoMF(conf, q.trainingData, q.testData)
    train, test = list(model.data.trainingData), list(model.data.testData)
    rec = dict(theta=[], beta=[], mu=[])
    update_expo = model._update_expo

    def spy_update_expo(X, n_users):
        update_expo(X, n_users)
        for k in rec:
            rec[k].append(getattr(model, k).copy())

    M.Parallel = sequential_parallel
    model._update_expo = spy_update_expo
    with contextlib.redirect_stdout(io.StringIO()):
        model.readConfiguration()
        model.initializing_log()
        model.initModel()
        theta0, beta0, mu0 = model.theta.copy(), model.beta.copy(), model.mu.copy()
        model.trainModel()
        model.evalRanking()
    measure = [m.strip() for m in model.measure]
    n_items = len(model.data.item)
    g = dict(seed=np.array(SEED), user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
             item_names=np.array([model.data.id2item[k] for k in range(n_items)]))
    t0, b0, m0 = EO.initial_state(g, model.emb_size)
    assert np.array_equal(theta0, t0) and np.array_equal(beta0, b0) and np.array_equal(mu0, m0)
    assert all(a.dtype == np.float32 for k in rec for a in rec[k])
    print('ExpoMF FilmTrust: users', len(g['user_names']), 'items', n_items, 'train', model.data.trainingSize(),
          '|theta|', float(np.abs(rec['theta'][-1]).max()), '|beta|', float(np.abs(rec['beta'][-1]).max()),
          'measure', measure)
    np.savez_compressed(
        os.path.join(OUT, 'expomf_filmtrust.npz'),
        train_users=np.array([e[0] for e in train]), train_items=np.array([e[1] for e in train]),
        train_rating=np.array([e[2] for e in train], dtype=np.float64),
        test_users=np.array([e[0] for e in test]), test_items=np.array([e[1] for e in test]),
        test_rating=np.array([e[2] for e in test], dtype=np.float64),
        theta_epoch=np.stack(rec['theta']), beta_epoch=np.stack(rec['beta']), mu_epoch=np.stack(rec['mu']),
        measure=np.array(measure), conf=np.array(CONF_EXPOMF), **g)


if __name__ == '__main__':
    _enter_workdir()
    gen_expomf()
