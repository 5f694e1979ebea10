#!/usr/bin/env python
"""Golden runs of the reference's SoRec and RSTE (model/rating/SoRec.py, model/rating/RSTE.py with
base/socialRecommender.py around them), UNMODIFIED.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose
module stubs and work-directory setup it shares: the GPU box never runs it.

FilmTrust trainset.txt / testset.txt with trust.txt (`-columns 0 1 2`), the shipped SoRec.conf / RSTE.conf
hyper-parameters, three epochs; SoRec runs at learning rate 0.01, because at SoRec.conf's 0.1 the reference's first
epoch (the user-sorted file order) overflows to NaN.  Recorded per run (tests/golden/sorec_filmtrust.npz, rste_filmtrust.npz):
  * the id maps, the training and test lists, and the cleaned relation list in order;
  * the MT19937 state before initModel and after every epoch's shuffle.  The visiting orders are not stored: the
    tests replay the shuffles from these states, and the generator checks that the replay gives the recorded orders;
  * the tables after epoch 1 (float32) and after the last epoch.  The initial tables are not stored: they come
    from the seed (oracle/sorec_rste_oracle.py: initial_tables), which the generator checks;
  * the losses and learning rates of every epoch, the epoch lines the model printed, each epoch's measure, the
    final measure and the raw test predictions.

Small constructed sets (CASES below), each run through the reference, go into tests/golden/social_rating_cases.npz
with their input files and outputs.  Together they hold a self-follow, a relation line listed twice with
different weights, followees whose weights are all zero, a followee who is not a training user, a user who follows
nobody, test lines with unknown users and items, a social file without a weight column, and an RSTE run with
item.ranking=on.

Usage:  python oracle/gen_golden_sorec_rste.py
"""
import contextlib
import importlib
import io
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen_golden import OUT, _enter_workdir, _state_to_array   # noqa: E402
from oracle import sorec_rste_oracle as SR                    # noqa: E402

CONF = """ratings=%(train)s
social=%(social)s
ratings.setup=-columns 0 1 2
social.setup=-columns %(cols)s
model.name=%(name)s
evaluation.setup=-testSet %(test)s
item.ranking=%(ranking)s -topN %(topn)s
num.factors=%(d)d
num.max.epoch=3
learnRate=-init %(lr)s -max 1
reg.lambda=-u %(ru)s -i %(ri)s -b 0.1 -s %(rs)s
%(name)s=%(extra)s
output.setup=on -dir ./results/
"""
FT = dict(train='./dataset/FilmTrust/trainset.txt', test='./dataset/FilmTrust/testset.txt',
          social='./dataset/FilmTrust/trust.txt', cols='0 1 2', ranking='off', topn='10')
SOREC = dict(name='SoRec', d=5, lr='0.01', ru='0.05', ri='0.05', rs='0.1', extra='-z 0.1')     # SoRec.conf, lr 0.01
RSTE = dict(name='RSTE', d=5, lr='0.01', ru='0.001', ri='0.001', rs='0.1', extra='-alpha 0.6')  # RSTE.conf
SEED = 11

# constructed social file: a self-follow (u1), a repeated line with a new weight (u2 -> u3), a followee who is not a
# training user (u3 -> u9), zero-weight followees (u4), and u8 follows nobody
SOCIAL_CASE = [('u1', 'u2', 0.8), ('u1', 'u1', 0.5), ('u2', 'u3', 0.4), ('u2', 'u3', 0.9), ('u3', 'u9', 1.0),
               ('u4', 'u5', 0.0), ('u4', 'u6', 0.0), ('u5', 'u1', 0.7), ('u6', 'u2', 0.3), ('u6', 'u7', 0.6),
               ('u7', 'u1', 1.0), ('u3', 'u5', 0.2)]
CASES = [  # (tag, model, weighted social file, item.ranking)
    ('sorec_w', SOREC, True, 'off'), ('rste_w', RSTE, True, 'off'), ('rste_rank', RSTE, True, 'on'),
    ('sorec_nw', SOREC, False, 'off'), ('rste_nw', RSTE, False, 'off')]


def _case_files():
    rs = np.random.RandomState(3)
    lines, seen = [], set()
    while len(lines) < 40:
        u, i = 'u%d' % rs.randint(1, 9), 'i%d' % rs.randint(1, 7)
        if (u, i) not in seen:
            seen.add((u, i))
            lines.append('%s %s %.1f' % (u, i, 0.5 * rs.randint(1, 9)))
    test = ['u1 i2 3.0', 'u99 i1 2.0', 'u3 i99 1.5', 'u98 i97 4.0', 'u4 i3 2.5', 'u8 i1 3.5', 'u6 i5 1.0',
            'u2 i6 2.0', 'u5 i4 3.0', 'u7 i2 0.5']
    files = {'case_train.txt': lines, 'case_test.txt': test,
             'case_social_w.txt': ['%s %s %s' % r for r in SOCIAL_CASE],
             'case_social_nw.txt': ['%s %s' % r[:2] for r in SOCIAL_CASE]}
    for name, body in files.items():
        with open(name, 'w') as f:
            f.write('\n'.join(body) + '\n')
    return {k: np.array(v) for k, v in files.items()}


def run(params, seed):
    from util.config import ModelConf
    from QRec import QRec
    name = params['name']
    text = CONF % params
    cname = '%s_golden.conf' % name
    with open(cname, 'w') as f:
        f.write(text)
    random.seed(seed)
    np.random.seed(seed)
    conf = ModelConf(cname)
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    cls = getattr(importlib.import_module('model.rating.' + name), name)
    model = cls(conf, q.trainingData, q.testData, q.relation)
    first = list(model.data.trainingData)
    where = {id(e): k for k, e in enumerate(first)}
    rec = dict(order=[], P=[], Q=[], Z=[], loss=[], lrate=[], states=[], measure=[])
    orig = cls.isConverged

    def spy(self, epoch):
        rec['order'].append(np.array([where[id(e)] for e in self.data.trainingData], dtype=np.int32))
        rec['P'].append(self.P.copy())
        rec['Q'].append(self.Q.copy())
        if hasattr(self, 'Z'):
            rec['Z'].append(self.Z.copy())
        rec['loss'].append(float(self.loss))
        before = self.lRate
        r = orig(self, epoch)
        rec['measure'].append([m.strip() for m in self.measure] if not self.ranking.isMainOn() else [])
        rec['lrate'].append((before, self.lRate))
        rec['states'].append(_state_to_array(random.getstate()))
        return r

    cls.isConverged = spy
    out = io.StringIO()
    try:
        with contextlib.redirect_stdout(out):
            model.readConfiguration()
            model.initializing_log()
            state_before = _state_to_array(random.getstate())
            model.initModel()
            init = dict(P0=model.P.copy(), Q0=model.Q.copy())
            if hasattr(model, 'Z'):
                init['Z0'] = model.Z.copy()
            model.trainModel()
            if model.ranking.isMainOn():
                model.evalRanking()
            else:
                model.evalRatings()
    finally:
        cls.isConverged = orig
    rel = model.social.relation
    lines = [ln for ln in out.getvalue().splitlines() if ' epoch ' in ln and 'loss = ' in ln]
    g = dict(user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
             item_names=np.array([model.data.id2item[k] for k in range(len(model.data.item))]),
             train_users=np.array([e[0] for e in first]), train_items=np.array([e[1] for e in first]),
             train_rating=np.array([e[2] for e in first], dtype=np.float64),
             test_users=np.array([e[0] for e in model.data.testData]),
             test_items=np.array([e[1] for e in model.data.testData]),
             test_rating=np.array([e[2] for e in model.data.testData], dtype=np.float64),
             rel_u1=np.array([r[0] for r in rel]), rel_u2=np.array([r[1] for r in rel]),
             rel_w=np.array([float(r[2]) for r in rel], dtype=np.float64),
             global_mean=np.array(model.data.globalMean), mt_state_before=state_before,
             mt_state_after_epoch=np.stack(rec['states']),
             P_epoch1=rec['P'][0].astype(np.float32), Q_epoch1=rec['Q'][0].astype(np.float32),
             P_last=rec['P'][-1], Q_last=rec['Q'][-1],
             loss=np.array(rec['loss']), lrate=np.array(rec['lrate']), epoch_lines=np.array(lines),
             epoch_measure=np.array(rec['measure']), measure=np.array([m.strip() for m in model.measure]),
             seed=np.array(seed), conf=np.array(text))
    for k, t in zip(('P0', 'Q0', 'Z0'), SR.initial_tables(seed, len(g['user_names']), len(g['item_names']),
                                                         params['d'], 'Z0' in init)):
        assert np.array_equal(t, init[k])
    if not model.ranking.isMainOn():
        g['test_pred'] = np.array([e[3] for e in model.data.testData], dtype=np.float64)
    if rec['Z']:
        g.update(Z_epoch1=rec['Z'][0].astype(np.float32), Z_last=rec['Z'][-1])
    print(name, params.get('train'), 'train', model.data.trainingSize(), 'relations', len(rel), 'losses', rec['loss'],
          'measure', g['measure'].tolist())
    for e, o in enumerate(_replayed_orders(len(first), state_before, len(rec['order']))):
        assert np.array_equal(o, rec['order'][e])
    return g


def _replayed_orders(n, state, epochs):
    """The visiting orders random.shuffle gives from the generator state `state` (file order first)."""
    rng = random.Random()
    rng.setstate((3, tuple(int(x) for x in state), None))
    order, out = list(range(n)), []
    for _ in range(epochs):
        out.append(np.array(order, np.int32))
        rng.shuffle(order)
    return out


def main():
    _enter_workdir()
    for params, fname in ((SOREC, 'sorec_filmtrust.npz'), (RSTE, 'rste_filmtrust.npz')):
        g = run(dict(FT, **params), SEED)
        np.savez_compressed(os.path.join(OUT, fname), **g)
    files = _case_files()
    cases = {}
    for tag, params, weighted, ranking in CASES:
        p = dict(params, train='case_train.txt', test='case_test.txt', topn='3', ranking=ranking,
                 social='case_social_w.txt' if weighted else 'case_social_nw.txt', cols='0 1 2' if weighted else '0 1',
                 lr='0.05')
        g = run(p, SEED + len(cases))
        cases.update({'%s/%s' % (tag, k): v for k, v in g.items()})
    cases.update({'files/%s' % k: v for k, v in files.items()})
    cases['tags'] = np.array([c[0] for c in CASES])
    np.savez_compressed(os.path.join(OUT, 'social_rating_cases.npz'), **cases)


if __name__ == '__main__':
    main()
