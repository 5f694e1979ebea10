#!/usr/bin/env python
"""Golden runs of the reference's memory-based rating models (model/rating/UserKNN.py, ItemKNN.py, SlopeOne.py),
UNMODIFIED, through its QRec driver.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose work-directory setup
it shares: the GPU box never runs it.

Recorded in tests/golden/knn_filmtrust.npz:
  * FilmTrust (trainset / testset): the training and test lists as the model holds them;
  * for UserKNN and ItemKNN with each of pcc, cos and euclidean (20 neighbours): the raw float64 prediction of every
    test line (the value predictForRating returns), the rating-prediction lines and the measure lines, and each
    query's first sorted entries (names and float64 similarities) -- 32 for pcc, 20 for cos and euclidean.  For pcc
    also the full sorted list of the first query, the last query, the first cold query (if any) and the query with the
    longest run of similarities tied with the 20th across the K boundary;
  * the same for SlopeOne (no lists);
  * small constructed sets (`case<n>_...`), each with cold test users and items, a repeated training line and stored
    ratings of -1, run for UserKNN and ItemKNN with pcc, cos, euclidean and 'foo' (which falls through to cosine) at
    num.neighbors -1, 0, 2 and 50 (past every list), and for SlopeOne: the training / test lists, and per run the raw
    predictions, the prediction and measure lines, or the exception the run raised (the last case is the first seed
    whose runs include a ZeroDivisionError) with the predictions made before it.

Usage:  python oracle/gen_golden_knn.py   (writes tests/golden/knn_filmtrust.npz)
"""
import contextlib
import glob
import io
import os
import random
import shutil
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import OUT, _enter_workdir   # noqa: E402

CONF = """ratings=%(train)s
ratings.setup=-columns 0 1 2
model.name=%(name)s
evaluation.setup=-testSet %(test)s
item.ranking=off -topN 10
similarity=%(sim)s
num.neighbors=%(k)d
output.setup=on -dir ./results/
"""
FT = dict(train='./dataset/FilmTrust/trainset.txt', test='./dataset/FilmTrust/testset.txt')
K = 20
CASE_SIMS = ('pcc', 'cos', 'euclidean', 'foo')
CASE_KS = (-1, 0, 2, 50)


def run(name, sim, k, paths):
    """One reference run: (model, raw predictions, prediction lines, measure lines, error name or '')."""
    import importlib
    from util.config import ModelConf
    from QRec import QRec
    shutil.rmtree('results', ignore_errors=True)
    os.makedirs('results')
    with open('run.conf', 'w') as f:
        f.write(CONF % dict(name=name, sim=sim, k=k, **paths))
    conf = ModelConf('run.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    cls = getattr(importlib.import_module('model.rating.' + name), name)
    model = cls(conf, q.trainingData, q.testData)
    raw = []
    orig = cls.predictForRating

    def spy(self, u, i):
        p = orig(self, u, i)
        raw.append(float(p))
        return p

    cls.predictForRating = spy
    error = ''
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            model.execute()
    except ZeroDivisionError as e:
        error = type(e).__name__
    finally:
        cls.predictForRating = orig
    lines, measure = [], []
    if not error:
        with open(glob.glob('results/*-rating-predictions*')[0]) as f:
            lines = [s.rstrip('\n') for s in f.readlines()[1:]]
        measure = [m.strip() for m in model.measure]
    return model, np.array(raw, dtype=np.float64), np.array(lines), np.array(measure), error


def lists(model):
    return getattr(model, 'topUsers', None) or getattr(model, 'topItems', None)


def head(top, queries, keep):
    names = np.array([[n for n, _ in top[q][:keep]] + [''] * (keep - len(top[q][:keep])) for q in queries])
    sims = np.array([[float(s) for _, s in top[q][:keep]] + [0.0] * (keep - len(top[q][:keep])) for q in queries])
    return names, sims


def filmtrust(arrays):
    for name in ('UserKNN', 'ItemKNN', 'SlopeOne'):
        for sim in (('pcc', 'cos', 'euclidean') if name != 'SlopeOne' else ('pcc',)):
            model, raw, lines, measure, error = run(name, sim, K, FT)
            assert not error
            tag = name if name == 'SlopeOne' else '%s_%s' % (name, sim)
            if 'train_users' not in arrays:
                train, test = model.data.trainingData, model.data.testData
                for key, rows in (('train', train), ('test', test)):
                    arrays[key + '_users'] = np.array([e[0] for e in rows])
                    arrays[key + '_items'] = np.array([e[1] for e in rows])
                    arrays[key + '_rating'] = np.array([e[2] for e in rows], dtype=np.float64)
            arrays[tag + '_raw'], arrays[tag + '_lines'], arrays[tag + '_measure'] = raw, lines, measure
            top = lists(model)
            if top is not None:
                queries = list(top)
                arrays[tag + '_queries'] = np.array(queries)
                arrays[tag + '_top_len'] = np.array([len(top[q]) for q in queries], dtype=np.int64)
                arrays[tag + '_top_names'], arrays[tag + '_top_sims'] = head(top, queries, 32 if sim == 'pcc' else K)
                if sim == 'pcc':
                    known = model.data.user if name == 'UserKNN' else model.data.item
                    cold = [q for q in queries if q not in known]

                    def tie_run(q):
                        s = [float(x) for _, x in top[q]]
                        return sum(x == s[K - 1] for x in s) if len(s) > K else 0
                    chosen = dict(first=queries[0], last=queries[-1], tie=max(queries, key=tie_run))
                    if cold:
                        chosen['cold'] = cold[0]
                    for key, q in chosen.items():
                        arrays['%s_full_%s_query' % (tag, key)] = np.array(q)
                        arrays['%s_full_%s_names' % (tag, key)] = np.array([n for n, _ in top[q]])
                        arrays['%s_full_%s_sims' % (tag, key)] = np.array([float(s) for _, s in top[q]])
            print(tag, 'measure', list(measure))


def constructed(seed):
    """A small training / test list: 9 users x 7 items, ratings with ties, stored -1s, one repeated training line;
    test lines of cold users and on cold items first (so that they are earlier queries of the warm ones), then of warm
    users on rated and unrated items."""
    rng = random.Random(seed)
    vals = (-1.0, 0.5, 1.0, 2.0, 2.0, 3.0, 4.0)
    train = []
    for u in range(9):
        for i in rng.sample(range(7), rng.randint(1, 5)):
            train.append(('u%d' % u, 'i%d' % i, rng.choice(vals)))
    u0, i0, _ = train[rng.randrange(len(train))]
    train.append((u0, i0, rng.choice(vals)))                     # repeated line: its last value counts
    test = [('cu0', 'i%d' % rng.randrange(7), 2.0), ('u%d' % rng.randrange(9), 'ci0', 2.0), ('cu1', 'ci1', 1.0)]
    test += [('u%d' % rng.randrange(9), 'i%d' % rng.randrange(7), 3.0) for _ in range(12)]   # after the cold ones
    seen, uniq = set(), []
    for t in test:                                               # one line per (user, item), as a test dict keeps
        if t[:2] not in seen:
            seen.add(t[:2])
            uniq.append(t)
    return train, uniq


def write(path, rows):
    with open(path, 'w') as f:
        for u, i, r in rows:
            f.write('%s %s %r\n' % (u, i, r))


def run_case(n, seed, arrays):
    train, test = constructed(seed)
    write('case_train.txt', train)
    write('case_test.txt', test)
    paths = dict(train='case_train.txt', test='case_test.txt')
    out = {'case%d_train_%s' % (n, k): np.array(v) for k, v in
           (('users', [t[0] for t in train]), ('items', [t[1] for t in train]))}
    out['case%d_train_rating' % n] = np.array([t[2] for t in train], dtype=np.float64)
    out['case%d_test_users' % n] = np.array([t[0] for t in test])
    out['case%d_test_items' % n] = np.array([t[1] for t in test])
    out['case%d_test_rating' % n] = np.array([t[2] for t in test], dtype=np.float64)
    errors = 0
    runs = [(name, sim, k) for name in ('UserKNN', 'ItemKNN') for sim in CASE_SIMS for k in CASE_KS]
    runs.append(('SlopeOne', 'pcc', 20))
    for name, sim, k in runs:
        _, raw, lines, measure, error = run(name, sim, k, paths)
        tag = 'case%d_%s_%s_%d' % (n, name, sim, k) if name != 'SlopeOne' else 'case%d_SlopeOne' % n
        out[tag + '_raw'], out[tag + '_lines'], out[tag + '_measure'] = raw, lines, measure
        out[tag + '_error'] = np.array(error)
        errors += bool(error)
    arrays.update(out)
    return errors


def main():
    _enter_workdir()
    arrays = {}
    filmtrust(arrays)
    n = 0
    for seed in (1, 2):
        run_case(n, seed, arrays)
        n += 1
    seed = 100
    while True:                                                  # the first seed with a ZeroDivisionError
        probe = {}
        if run_case(n, seed, probe):
            arrays.update(probe)
            break
        seed += 1
    arrays['case_seeds'] = np.array([1, 2, seed])
    arrays['case_sims'], arrays['case_ks'] = np.array(CASE_SIMS), np.array(CASE_KS)
    arrays['conf'] = np.array(CONF)
    print('cases: seeds', [1, 2, seed], 'errors in the last:',
          [k for k, v in arrays.items() if k.startswith('case%d_' % n) and k.endswith('_error') and str(v)])
    np.savez_compressed(os.path.join(OUT, 'knn_filmtrust.npz'), **arrays)


if __name__ == '__main__':
    main()
