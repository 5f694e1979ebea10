#!/usr/bin/env python
"""Golden runs of the reference's EE and SREE (model/rating/EE.py, model/rating/SREE.py), UNMODIFIED.  TEST
INFRASTRUCTURE ONLY, like oracle/gen_golden_socialmf_soreg.py, whose constructed data it shares: the GPU box never
runs it.

FilmTrust trainset.txt / testset.txt (with trust.txt for SREE), the shipped EE.conf / SREE.conf hyper-parameters and
their regB (`-b`), three epochs, seed 11 (tests/golden/ee_filmtrust.npz, sree_filmtrust.npz).  Each run records what
oracle/gen_golden_sorec_rste.py's `run` records (id maps, lists, generator states, tables after epoch 1 as float32 and
after the last epoch, losses, learning rates, epoch lines, measures, raw test predictions), and also:
  * Bu0 / Bi0, the biases initModel drew, and the biases after epoch 1 (float32) and after the last epoch;
  * for SREE, the relation list as read (raw_u1 / raw_u2 / raw_w) and social.user, its first-appearance order.
The SREE run with `item.ranking=on -topN 10` trains exactly as the rating run (ranking consumes no random draws), so
only its configuration, epoch lines, ranking measure and recommendation lists are kept (sree_filmtrust.npz, rank_*;
rank_rec_items holds each recommendation line without its scores).  sree_filmtrust.npz leaves out the id maps and the
training and test lists, which are those of ee_filmtrust.npz.

Constructed runs (tests/golden/ee_sree_cases.npz) use the training, test and social files of
gen_golden_socialmf_soreg.py: a mutual follow with a different weight each way, a self-follow, a zero-weight followee,
a followee visited after its follower (u3 -> u5) and one visited before (u7 -> u3), relation ends that are not training
users (u9 first in social.user, u99), a training user absent from the social file (u8), and test lines with an unknown
user and an unknown item.  SREE runs on it with and without the weight column; EE runs on the ratings alone.

Usage:  python oracle/gen_golden_ee_sree.py
"""
import contextlib
import importlib
import io
import os
import random
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen_golden import OUT, _enter_workdir, _state_to_array   # noqa: E402
import gen_golden_socialmf_soreg as GM                        # noqa: E402
import gen_golden_sorec_rste as GS                            # noqa: E402
from oracle import ee_sree_oracle as EO                       # noqa: E402
from oracle import sorec_rste_oracle as SR                    # noqa: E402

CONF = """ratings=%(train)s
%(social_lines)sratings.setup=-columns 0 1 2
model.name=%(name)s
evaluation.setup=-testSet %(test)s
item.ranking=%(ranking)s -topN %(topn)s
num.factors=%(d)d
num.max.epoch=3
learnRate=-init %(lr)s -max 1
reg.lambda=-u %(ru)s -i %(ri)s -b %(rb)s -s 0.1
%(extra)soutput.setup=on -dir ./results/
"""
EE = dict(name='EE', d=10, lr='0.005', ru='0.005', ri='0.005', rb='0.005', extra='', social=None)          # EE.conf
SREE = dict(name='SREE', d=10, lr='0.01', ru='0.01', ri='0.01', rb='0.01', extra='SREE=-alpha 0.5\n',       # SREE.conf
            social='./dataset/FilmTrust/trust.txt')
FT = dict(train='./dataset/FilmTrust/trainset.txt', test='./dataset/FilmTrust/testset.txt', ranking='off', topn='10',
          cols='0 1 2')
SEED = 11
LISTS = ('user_names', 'item_names', 'train_users', 'train_items', 'train_rating', 'test_users', 'test_items',
         'test_rating')
CASES = [('ee', EE, None), ('sree_w', SREE, True), ('sree_nw', SREE, False)]


def rec_items(line):
    """A recommendation line 'user: (item,score)* ...' without its scores: 'user: item* ...'."""
    return line.split(':')[0] + ':' + ''.join(' ' + a + b for a, b in re.findall(r'\(([^,]+),[^)]*\)(\*?)', line))


def run(params, seed):
    from util.config import ModelConf
    from util.io import FileIO
    from QRec import QRec
    name = params['name']
    social = params['social']
    text = CONF % dict(params, social_lines='' if social is None else
                       'social=%s\nsocial.setup=-columns %s\n' % (social, params['cols']))
    cname = '%s_golden.conf' % name
    with open(cname, 'w') as f:
        f.write(text)
    random.seed(seed)
    np.random.seed(seed)
    conf = ModelConf(cname)
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    cls = getattr(importlib.import_module('model.rating.' + name), name)
    model = (cls(conf, q.trainingData, q.testData) if social is None else
             cls(conf, q.trainingData, q.testData, q.relation))
    first = list(model.data.trainingData)
    where = {id(e): k for k, e in enumerate(first)}
    rec = dict(order=[], P=[], Q=[], Bu=[], Bi=[], loss=[], lrate=[], states=[], measure=[])
    orig = cls.isConverged

    def spy(self, epoch):
        rec['order'].append(np.array([where[id(e)] for e in self.data.trainingData], dtype=np.int32))
        for k in ('P', 'Q', 'Bu', 'Bi'):
            rec[k].append(getattr(self, k).copy())
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
            init = dict(P0=model.P.copy(), Q0=model.Q.copy(), Bu0=model.Bu.copy(), Bi0=model.Bi.copy())
            model.trainModel()
            if model.ranking.isMainOn():
                model.evalRanking()
            else:
                model.evalRatings()
    finally:
        cls.isConverged = orig
    lines = [ln for ln in out.getvalue().splitlines() if ' epoch ' in ln and 'loss = ' in ln]
    g = dict(user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
             item_names=np.array([model.data.id2item[k] for k in range(len(model.data.item))]),
             train_users=np.array([e[0] for e in first]), train_items=np.array([e[1] for e in first]),
             train_rating=np.array([e[2] for e in first], dtype=np.float64),
             test_users=np.array([e[0] for e in model.data.testData]),
             test_items=np.array([e[1] for e in model.data.testData]),
             test_rating=np.array([e[2] for e in model.data.testData], dtype=np.float64),
             global_mean=np.array(model.data.globalMean), mt_state_before=state_before,
             mt_state_after_epoch=np.stack(rec['states']), Bu0=init['Bu0'], Bi0=init['Bi0'],
             loss=np.array(rec['loss']), lrate=np.array(rec['lrate']), epoch_lines=np.array(lines),
             epoch_measure=np.array(rec['measure']), measure=np.array([m.strip() for m in model.measure]),
             seed=np.array(seed), conf=np.array(text))
    for k in ('P', 'Q', 'Bu', 'Bi'):
        g[k + '_epoch1'] = rec[k][0].astype(np.float32)
        g[k + '_last'] = rec[k][-1]
    if model.ranking.isMainOn():
        g['rec_items'] = np.array([rec_items(ln) for ln in model.recOutput[1:]])
    else:
        g['test_pred'] = np.array([e[3] for e in model.data.testData], dtype=np.float64)
    if social is not None:
        raw = FileIO.loadRelationship(conf, social)
        g.update(raw_u1=np.array([r[0] for r in raw]), raw_u2=np.array([r[1] for r in raw]),
                 raw_w=np.array([float(r[2]) for r in raw], dtype=np.float64),
                 social_user=np.array(list(model.social.user)))
    U, I, d = len(g['user_names']), len(g['item_names']), params['d']
    for k, t in zip(('P0', 'Q0'), SR.initial_tables(seed, U, I, d, False)):
        assert np.array_equal(t, init[k])
    for k, t in zip(('Bu0', 'Bi0'), EO.initial_biases(seed, U, I, d)):
        assert np.array_equal(t, init[k])
    print(name, params.get('train'), 'train', model.data.trainingSize(), 'losses', rec['loss'],
          'measure', g['measure'].tolist())
    for e, o in enumerate(GS._replayed_orders(len(first), state_before, len(rec['order']))):
        assert np.array_equal(o, rec['order'][e])
    return g


def main():
    _enter_workdir()
    ee = run(dict(FT, **EE), SEED)
    np.savez_compressed(os.path.join(OUT, 'ee_filmtrust.npz'), **ee)
    g = run(dict(FT, **SREE), SEED)
    r = run(dict(FT, **dict(SREE, ranking='on')), SEED)
    for k in ('P', 'Q', 'Bu', 'Bi'):
        assert np.array_equal(r[k + '_last'], g[k + '_last'])
    g.update({'rank_' + k: r[k] for k in ('conf', 'epoch_lines', 'measure', 'rec_items')})
    for k in LISTS:
        assert np.array_equal(g.pop(k), ee[k])
    np.savez_compressed(os.path.join(OUT, 'sree_filmtrust.npz'), **g)
    files = GM._case_files()
    cases = {}
    for k, (tag, params, weighted) in enumerate(CASES):
        p = dict(params, train='case_train.txt', test='case_test.txt', topn='3', ranking='off', lr='0.05',
                 cols='0 1 2' if weighted is not False else '0 1')
        if params['social'] is not None:
            p['social'] = 'case_social_w.txt' if weighted else 'case_social_nw.txt'
        g = run(p, SEED + k)
        cases.update({'%s/%s' % (tag, key): v for key, v in g.items()})
    cases.update({'files/%s' % key: v for key, v in files.items()})
    cases['tags'] = np.array([c[0] for c in CASES])
    np.savez_compressed(os.path.join(OUT, 'ee_sree_cases.npz'), **cases)


if __name__ == '__main__':
    main()
