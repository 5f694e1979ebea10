#!/usr/bin/env python
"""Golden runs of the reference's SocialMF and SoReg (model/rating/SocialMF.py, model/rating/SoReg.py with
base/socialRecommender.py around them), UNMODIFIED.  TEST INFRASTRUCTURE ONLY, like oracle/gen_golden_sorec_rste.py,
whose `run` records every run here: the GPU box never runs it.

FilmTrust trainset.txt / testset.txt with trust.txt (`-columns 0 1 2`), the shipped SocialMF.conf / SoReg.conf
hyper-parameters (learning rate 0.05), three epochs, seed 11 (tests/golden/socialmf_filmtrust.npz, soreg_filmtrust.npz).
On top of what `run` records (see gen_golden_sorec_rste.py), each run here holds:
  * the relation list as read, before the cleaning (raw_u1 / raw_u2 / raw_w): the user pass visits `social.user`, its
    first-appearance order;
  * social_user: that order, as the reference built it;
  * for SoReg, its similarities as (sim_user, sim_friend, sim_value) arrays in the order initModel computed them.

Small constructed sets (CASE_* below), each run through the reference, go into tests/golden/socialmf_soreg_cases.npz
with their input files and outputs.  Their social file holds a mutual follow with a different weight in each
direction, a user whose ratings are all equal and a trust pair with no co-rated item (the two degenerate Pearson
branches), zero-weight followees, a self-follow, relation ends that are not training users (one of them first in
`social.user`), and a training user absent from the social file; each model runs on it with and without the weight
column.

Usage:  python oracle/gen_golden_socialmf_soreg.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen_golden import OUT, _enter_workdir                    # noqa: E402
import gen_golden_sorec_rste as GS                            # noqa: E402

FT = GS.FT
SOCIALMF = dict(name='SocialMF', d=5, lr='0.05', ru='0.05', ri='0.05', rs='0.1', extra='')             # SocialMF.conf
SOREG = dict(name='SoReg', d=10, lr='0.05', ru='0.02', ri='0.02', rs='0.02', extra='-alpha 0.1')       # SoReg.conf
SEED = 11

CASE_TRAIN = {  # u5 rates everything 3.0 (zero variance); u6 shares no item with u1; u8 is not in the social file
    'u1': [('i1', 4.0), ('i2', 3.0), ('i3', 2.5), ('i4', 1.0)],
    'u2': [('i1', 3.5), ('i2', 2.0), ('i5', 4.0), ('i6', 1.5)],
    'u3': [('i2', 1.0), ('i3', 4.0), ('i4', 3.0), ('i7', 2.0)],
    'u4': [('i1', 2.0), ('i5', 3.5), ('i8', 4.0)],
    'u5': [('i2', 3.0), ('i3', 3.0), ('i6', 3.0)],
    'u6': [('i7', 4.0), ('i8', 1.5)],
    'u7': [('i1', 1.0), ('i4', 4.0), ('i6', 2.5), ('i8', 3.0)],
    'u8': [('i3', 2.0), ('i5', 1.0), ('i7', 3.5)],
}
CASE_SOCIAL = [('u9', 'u3', 1.0),                      # u9 is no training user, yet first in social.user
               ('u1', 'u2', 0.8), ('u2', 'u1', 0.3),   # mutual, a different weight each way
               ('u1', 'u1', 0.5),                      # self-follow
               ('u3', 'u5', 0.6),                      # u5's ratings are all equal
               ('u6', 'u1', 0.9),                      # no co-rated item
               ('u4', 'u5', 0.0), ('u4', 'u6', 0.0),   # followee weights summing to 0
               ('u5', 'u7', 0.4), ('u7', 'u3', 1.0), ('u2', 'u6', 0.2),
               ('u3', 'u99', 0.7),                     # a followee who is no training user
               ('u7', 'u2', 0.5)]
CASES = [('socialmf_w', SOCIALMF, True), ('soreg_w', SOREG, True), ('socialmf_nw', SOCIALMF, False),
         ('soreg_nw', SOREG, False)]


def _case_files():
    lines = ['%s %s %.1f' % (u, i, r) for u, row in CASE_TRAIN.items() for i, r in row]
    order = np.random.RandomState(5).permutation(len(lines))
    test = ['u1 i5 3.0', 'u99 i1 2.0', 'u3 i99 1.5', 'u5 i1 2.5', 'u6 i2 1.0', 'u8 i4 3.5', 'u4 i6 2.0',
            'u2 i7 4.0', 'u7 i3 0.5']
    files = {'case_train.txt': [lines[k] for k in order], 'case_test.txt': test,
             'case_social_w.txt': ['%s %s %s' % r for r in CASE_SOCIAL],
             'case_social_nw.txt': ['%s %s' % r[:2] for r in CASE_SOCIAL]}
    for name, body in files.items():
        with open(name, 'w') as f:
            f.write('\n'.join(body) + '\n')
    return {k: np.array(v) for k, v in files.items()}


def run(params, seed):
    """GS.run, plus the relation list as read, social.user and SoReg's similarities."""
    import importlib
    from util.config import ModelConf
    from util.io import FileIO
    name = params['name']
    cls = getattr(importlib.import_module('model.rating.' + name), name)
    seen = {}
    orig = cls.initModel

    def spy(self):
        orig(self)
        seen['user'] = list(self.social.user)
        if hasattr(self, 'Sim'):
            seen['sim'] = [(a, b, v) for a in self.Sim for b, v in self.Sim[a].items()]

    cls.initModel = spy
    try:
        g = GS.run(params, seed)
    finally:
        cls.initModel = orig
    raw = FileIO.loadRelationship(ModelConf('%s_golden.conf' % name), params['social'])
    g.update(raw_u1=np.array([r[0] for r in raw]), raw_u2=np.array([r[1] for r in raw]),
             raw_w=np.array([float(r[2]) for r in raw], dtype=np.float64), social_user=np.array(seen['user']))
    if 'sim' in seen:
        g.update(sim_user=np.array([s[0] for s in seen['sim']]), sim_friend=np.array([s[1] for s in seen['sim']]),
                 sim_value=np.array([s[2] for s in seen['sim']], dtype=np.float64))
    return g


def main():
    _enter_workdir()
    for params, fname in ((SOCIALMF, 'socialmf_filmtrust.npz'), (SOREG, 'soreg_filmtrust.npz')):
        g = run(dict(FT, **params), SEED)
        np.savez_compressed(os.path.join(OUT, fname), **g)
    files = _case_files()
    cases = {}
    for k, (tag, params, weighted) in enumerate(CASES):
        p = dict(params, train='case_train.txt', test='case_test.txt', topn='3', ranking='off',
                 social='case_social_w.txt' if weighted else 'case_social_nw.txt', cols='0 1 2' if weighted else '0 1')
        g = run(p, SEED + k)
        cases.update({'%s/%s' % (tag, key): v for key, v in g.items()})
    cases.update({'files/%s' % key: v for key, v in files.items()})
    cases['tags'] = np.array([c[0] for c in CASES])
    np.savez_compressed(os.path.join(OUT, 'socialmf_soreg_cases.npz'), **cases)


if __name__ == '__main__':
    main()
