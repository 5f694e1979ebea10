#!/usr/bin/env python
"""Golden run of the reference's SERec (model/ranking/SERec.py with base/socialRecommender.py around it), UNMODIFIED,
through its QRec driver on FilmTrust with its trust network.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py,
whose work-directory setup it shares: the GPU box never runs it.

Two things are swapped in the model's module namespace, neither changing what it computes:
  * `joblib.Parallel` becomes a sequential call (as in gen_golden_expomf.py), so that no worker processes are spawned;
    the batches it hands out are independent (every row reads only the old tables);
  * `np` becomes a proxy of numpy whose `tile` records its argument: the exact summed posteriors A of every epoch
    (`_update_expo` tiles A into a U x I matrix before forming the prior).

Recorded in tests/golden/serec_filmtrust.npz:
  * the training / test lists as the model holds them, the relation list as loaded, and the id maps;
  * theta and beta after every epoch (float32, as the reference keeps them).  The initial state is not stored: it
    comes from the seeded legacy numpy stream (oracle/serec_oracle.py: initial_state), which the generator checks;
  * A of every epoch (float64), and the degrees of T's rows, which the generator checks against the oracle's;
  * mu after every epoch for a few users -- the first of degree 0, the first of degree 1, the first of the largest
    degree and the three first and three last users (the ones numpy's summary prints) -- at every eighth item and the
    three first and three last items (a sample, to keep the file small; the prints cover the edges too);
  * the text of every epoch's `print(self.mu)` and the final measure lines.

Usage:  python oracle/gen_golden_serec.py   (writes tests/golden/serec_filmtrust.npz)
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
from gen_golden_expomf import sequential_parallel   # noqa: E402
from oracle import serec_oracle as SO        # noqa: E402

CONF_SEREC = """ratings=./dataset/FilmTrust/trainset.txt
social=./dataset/FilmTrust/trust.txt
ratings.setup=-columns 0 1 2
social.setup=-columns 0 1
model.name=SERec
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt
item.ranking=on -topN 10
num.factors=20
num.max.epoch=3
learnRate=-init 0.01 -max 1
reg.lambda=-u 1 -i 0.02 -b 0.02 -s 0.01
output.setup=on -dir ./results/
"""
SEED = 5


class TileRecorder(object):
    """numpy, except that `tile` also keeps a copy of the array it tiles."""

    def __init__(self, log):
        self._log = log

    def __getattr__(self, name):
        return getattr(np, name)

    def tile(self, A, reps):
        self._log.append(np.array(A, dtype=np.float64, copy=True))
        return np.tile(A, reps)


def gen_serec():
    from util.config import ModelConf
    from QRec import QRec
    import model.ranking.SERec as M
    with open('SERec_ft.conf', 'w') as f:
        f.write(CONF_SEREC)
    random.seed(SEED)
    np.random.seed(SEED)
    conf = ModelConf('SERec_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    relation = [list(r) for r in q.relation]
    model = M.SERec(conf, q.trainingData, q.testData, q.relation)
    train, test = list(model.data.trainingData), list(model.data.testData)
    asums = []
    rec = dict(theta=[], beta=[], mu_rows=[], mu_str=[])
    watch, items = [], []
    update_expo = model._update_expo

    def spy_update_expo(X, n_users):
        rec['mu_str'].append(str(model.mu))          # what _update has just printed
        update_expo(X, n_users)
        if not watch:
            deg = np.asarray(model.T.sum(axis=1)).ravel()
            U = len(deg)
            first = [int(np.flatnonzero(deg == 0)[0]), int(np.flatnonzero(deg == 1)[0]), int(np.argmax(deg))]
            watch.extend(first + [u for u in (0, 1, 2, U - 3, U - 2, U - 1) if u not in first])
            I = model.num_items
            items.extend(sorted(set(range(0, I, 8)) | {0, 1, 2, I - 3, I - 2, I - 1}))
        rec['theta'].append(model.theta.copy())
        rec['beta'].append(model.beta.copy())
        rec['mu_rows'].append(np.asarray(model.mu)[np.ix_(watch, items)].copy())

    M.Parallel = sequential_parallel
    M.np = TileRecorder(asums)
    model._update_expo = spy_update_expo
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        model.readConfiguration()
        model.initializing_log()
        model.initModel()
        theta0, beta0 = model.theta.copy(), model.beta.copy()
        model.trainModel()
    with contextlib.redirect_stdout(io.StringIO()):
        model.evalRanking()
    measure = [m.strip() for m in model.measure]
    n_items = len(model.data.item)
    g = dict(seed=np.array(SEED), user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
             item_names=np.array([model.data.id2item[k] for k in range(n_items)]))
    t0, b0 = SO.initial_state(g, model.emb_size)
    assert np.array_equal(theta0, t0) and np.array_equal(beta0, b0)
    deg = np.asarray(model.T.sum(axis=1)).ravel().astype(np.int32)
    assert np.array_equal(deg, SO.degrees(g['user_names'], relation))
    assert len(asums) == len(rec['theta']) and all(a.shape == (n_items,) for a in asums)
    assert all(a.dtype == np.float32 for k in ('theta', 'beta') for a in rec[k])
    text = out.getvalue()
    assert all(s + '\n' in text for s in rec['mu_str'])
    print('SERec FilmTrust: users', len(g['user_names']), 'items', n_items, 'train', model.data.trainingSize(),
          'relations', len(relation), 'deg: zero', int((deg == 0).sum()), 'max', int(deg.max()), 'watched', watch,
          '|theta|', float(np.abs(rec['theta'][-1]).max()), '|beta|', float(np.abs(rec['beta'][-1]).max()),
          'measure', measure)
    np.savez_compressed(
        os.path.join(OUT, 'serec_filmtrust.npz'),
        train_users=np.array([e[0] for e in train]), train_items=np.array([e[1] for e in train]),
        train_rating=np.array([e[2] for e in train], dtype=np.float64),
        test_users=np.array([e[0] for e in test]), test_items=np.array([e[1] for e in test]),
        test_rating=np.array([e[2] for e in test], dtype=np.float64),
        rel_u1=np.array([r[0] for r in relation]), rel_u2=np.array([r[1] for r in relation]),
        rel_w=np.array([r[2] for r in relation], dtype=np.float64), deg=deg,
        theta_epoch=np.stack(rec['theta']), beta_epoch=np.stack(rec['beta']), asum_epoch=np.stack(asums),
        mu_users=np.array(watch, dtype=np.int64), mu_items=np.array(items, dtype=np.int64), mu_rows_epoch=np.stack(rec['mu_rows']),
        mu_str=np.array(rec['mu_str']), measure=np.array(measure), conf=np.array(CONF_SEREC), **g)


if __name__ == '__main__':
    _enter_workdir()
    gen_serec()
