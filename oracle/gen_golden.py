#!/usr/bin/env python
"""Golden-vector generator: runs the UNMODIFIED reference (Coder-Yu/QRec, mounted
read-only at /root/reference) in this container and records what the hot path
consumed and produced.  TEST INFRASTRUCTURE ONLY -- nothing in the product path
imports this file; the GPU box never runs it (there is no /root/reference there).

What is exercised (reference file:line):
  * QRec.__init__            QRec.py:8-47        load FilmTrust, `-ap 0.2 -b 1` split
  * Rating.__generateSet     data/rating.py:33-67   first-appearance id maps
  * IterativeRecommender.initModel  base/iterativeRecommender.py:36-39
  * BPR.trainModel / optimization   model/ranking/BPR.py:19-53   (numpy float64 SGD)
  * IterativeRecommender.isConverged / updateLearningRate  base/iterativeRecommender.py:56-63,82-102
  * Recommender.evalRanking  base/recommender.py:127-179
  * DeepRecommender.next_batch_pairwise / next_batch_pointwise  base/deepRecommender.py:29-77
  * GraphRecommender.create_joint_sparse_adjaceny / create_sparse_rating_matrix
                              base/graphRecommender.py:10-29,41-51
  * BasicMF / PMF / SVD .trainModel   model/rating/BasicMF.py:9-25, PMF.py:9-28, SVD.py:9-36
    (pointwise sequential SGD; §8 f-4), with the per-epoch shuffle of isConverged and the
    MAE / RMSE of evalRatings (base/recommender.py:95-125, util/measure.py)
  * SBPR.initModel / next_batch   model/ranking/SBPR.py:12-29, 69-101 (social-feedback sets, minibatch sampler)

`tensorflow` and `mkl` are absent from this image; both are stubbed with empty
modules because the reference imports them at module level (model/ranking/BPR.py:7,
QRec.py:6).  The numpy path never calls into either.

Usage:  python oracle/gen_golden.py [bpr] [mf] [sbpr] [reference]   (default: all sections; writes tests/golden/)
"""
import os
import sys
import types
import random
import tempfile
import contextlib
import io

import numpy as np

REF = '/root/reference'
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(REPO, 'tests', 'golden')

CONF_BPR = """ratings=./dataset/FilmTrust/ratings.txt
ratings.setup=-columns 0 1 2
model.name=BPR
evaluation.setup=-ap 0.2 -b 1
item.ranking=on -topN 10
num.factors=64
num.max.epoch=3
batch_size=2048
learnRate=-init 0.01 -max 1
reg.lambda=-u 0.001 -i 0.001 -b 0.2 -s 0.2
output.setup=on -dir ./results/
"""

CONF_LGCN = """ratings=./dataset/FilmTrust/ratings.txt
ratings.setup=-columns 0 1 2
model.name=LightGCN
evaluation.setup=-ap 0.2 -b 1
item.ranking=on -topN 10
num.factors=64
num.max.epoch=2
batch_size=2048
learnRate=-init 0.001 -max 1
LightGCN=-n_layer 3
reg.lambda=-u 0.001 -i 0.001 -b 0.2 -s 0.2
output.setup=on -dir ./results/
"""

CONF_MF = """ratings=./dataset/FilmTrust/trainset.txt
ratings.setup=-columns 0 1 2
model.name=%(name)s
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt
item.ranking=off -topN 10
num.factors=%(d)d
num.max.epoch=3
batch_size=1024
learnRate=-init %(lr)s -max 1
reg.lambda=-u 0.01 -i 0.02 -b 0.03 -s 0.1
output.setup=on -dir ./results/
"""
MF_RUNS = (('BasicMF', 20, '0.03', 11), ('PMF', 10, '0.02', 12), ('SVD', 20, '0.005', 13))   # name, d, lr, seed


def _stub_modules():
    sys.modules.setdefault('tensorflow', types.ModuleType('tensorflow'))
    mkl = types.ModuleType('mkl')
    mkl.set_num_threads = lambda n: None
    mkl.get_max_threads = lambda: 1
    sys.modules.setdefault('mkl', mkl)


def _state_to_array(state):
    """random.getstate() -> uint32[625] (624 words + index)."""
    version, internal, gauss = state
    assert version == 3 and gauss is None
    return np.array(internal, dtype=np.uint32)


def _enter_workdir():
    assert os.path.isdir(REF), 'reference checkout not mounted'
    _stub_modules()
    sys.path.insert(0, REF)
    work = tempfile.mkdtemp(prefix='qrec_golden_')
    os.chdir(work)
    os.symlink(os.path.join(REF, 'dataset'), 'dataset')
    os.makedirs('log', exist_ok=True)
    os.makedirs('results', exist_ok=True)


def gen_bpr():
    with open('BPR_ft.conf', 'w') as f:
        f.write(CONF_BPR)
    with open('LGCN_ft.conf', 'w') as f:
        f.write(CONF_LGCN)

    from util.config import ModelConf
    from QRec import QRec
    from model.ranking.BPR import BPR

    # ------------------------------------------------------------------ BPR numpy path
    random.seed(0)
    np.random.seed(0)
    conf = ModelConf('BPR_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(conf)
    train, test = q.trainingData, q.testData
    state_after_split = _state_to_array(random.getstate())

    model = BPR(conf, train, test)
    # training list exactly as the model holds it at construction (data/rating.py:27)
    train_users = np.array([e[0] for e in model.data.trainingData])
    train_items = np.array([e[1] for e in model.data.trainingData])
    train_rating = np.array([e[2] for e in model.data.trainingData], dtype=np.float64)
    test_users = np.array([e[0] for e in model.data.testData])
    test_items = np.array([e[1] for e in model.data.testData])
    test_rating = np.array([e[2] for e in model.data.testData], dtype=np.float64)
    user_names = np.array([model.data.id2user[k] for k in range(len(model.data.user))])
    item_names = np.array([model.data.id2item[k] for k in range(len(model.data.item))])

    rec = dict(triples=[], cur=[], P=[], Q=[], loss=[], lrate=[], states=[])
    orig_opt = BPR.optimization
    orig_conv = BPR.isConverged

    def spy_opt(self, u, i, j):
        rec['cur'].append((u, i, j))
        return orig_opt(self, u, i, j)

    def spy_conv(self, epoch):
        rec['triples'].append(np.array(rec['cur'], dtype=np.int32))
        rec['cur'] = []
        rec['P'].append(self.P.copy())
        rec['Q'].append(self.Q.copy())
        rec['loss'].append(float(self.loss))
        lr_before = self.lRate
        r = orig_conv(self, epoch)
        rec['lrate'].append((lr_before, self.lRate))
        rec['states'].append(_state_to_array(random.getstate()))
        return r

    BPR.optimization = spy_opt
    BPR.isConverged = spy_conv
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            model.readConfiguration()
            model.initializing_log()
            state_before_init = _state_to_array(random.getstate())
            model.initModel()
            P0, Q0 = model.P.copy(), model.Q.copy()
            model.trainModel()
            model.evalRanking()
    finally:
        BPR.optimization = orig_opt
        BPR.isConverged = orig_conv
    measure = [m.strip() for m in model.measure]
    print('BPR FilmTrust: train', model.data.trainingSize(), 'losses', rec['loss'], 'measure', measure)

    # check the regenerable init: legacy numpy stream is stable across versions
    np.random.seed(0)
    P0r = np.random.rand(len(model.data.user), 64) / 3
    Q0r = np.random.rand(len(model.data.item), 64) / 3
    assert np.array_equal(P0r, P0) and np.array_equal(Q0r, Q0)
    assert np.array_equal(state_before_init, state_after_split)

    # top-10 recommendation lists (ids) for the first 64 test users, for the eval parity test
    rec_lines = model.recOutput[1:65]

    np.savez_compressed(
        os.path.join(OUT, 'bpr_filmtrust_seed0.npz'),
        user_names=user_names, item_names=item_names,
        train_users=train_users, train_items=train_items, train_rating=train_rating,
        test_users=test_users, test_items=test_items, test_rating=test_rating,
        mt_state_after_split=state_after_split,
        mt_state_after_epoch=np.stack(rec['states']),
        triples_epoch=np.stack(rec['triples']),            # [3, n, 3] int32 (u,i,j) in reference order
        P_epoch1=rec['P'][0], Q_epoch1=rec['Q'][0],        # float64
        P_epoch3=rec['P'][2].astype(np.float32), Q_epoch3=rec['Q'][2].astype(np.float32),
        loss=np.array(rec['loss']), lrate=np.array(rec['lrate']),
        measure=np.array(measure), rec_lines=np.array(rec_lines),
        conf=np.array(CONF_BPR),
    )

    # ------------------------------------------------------------------ samplers (TF-style path)
    from base.deepRecommender import DeepRecommender
    from base.graphRecommender import GraphRecommender
    random.seed(1234)
    np.random.seed(1234)
    lconf = ModelConf('LGCN_ft.conf')
    with contextlib.redirect_stdout(io.StringIO()):
        q2 = QRec(lconf)
    g = GraphRecommender(lconf, q2.trainingData, q2.testData)
    with contextlib.redirect_stdout(io.StringIO()):
        g.readConfiguration()
    g_train_users = np.array([e[0] for e in g.data.trainingData])
    g_train_items = np.array([e[1] for e in g.data.trainingData])
    g_user_names = np.array([g.data.id2user[k] for k in range(len(g.data.user))])
    g_item_names = np.array([g.data.id2item[k] for k in range(len(g.data.item))])
    st_pair = _state_to_array(random.getstate())
    pair_batches = [np.array(b, dtype=np.int32) for b in DeepRecommender.next_batch_pairwise(g)]
    st_after_pair = _state_to_array(random.getstate())
    # the list was shuffled in place by the generator; record the new order as (u,i) ids
    shuffled_u = np.array([g.data.user[e[0]] for e in g.data.trainingData], dtype=np.int32)
    shuffled_i = np.array([g.data.item[e[1]] for e in g.data.trainingData], dtype=np.int32)
    st_point = _state_to_array(random.getstate())
    point_batches = []
    for n, b in enumerate(DeepRecommender.next_batch_pointwise(g)):
        point_batches.append(np.array(b, dtype=np.int32))
        if n == 1:
            break
    st_after_point = _state_to_array(random.getstate())

    adj = g.create_joint_sparse_adjaceny().tocsr()
    adj.sort_indices()
    rmat = g.create_sparse_rating_matrix().tocsr()
    rmat.sort_indices()
    np.savez_compressed(
        os.path.join(OUT, 'sampler_graph_filmtrust_seed1234.npz'),
        user_names=g_user_names, item_names=g_item_names,
        train_users=g_train_users, train_items=g_train_items,
        mt_state_before_pairwise=st_pair, mt_state_after_pairwise=st_after_pair,
        pair_first=pair_batches[0], pair_last=pair_batches[-1],
        pair_all_j=np.concatenate([b[2] for b in pair_batches]),
        pair_num_batches=np.array(len(pair_batches)),
        shuffled_u=shuffled_u, shuffled_i=shuffled_i,
        mt_state_before_pointwise=st_point, mt_state_after_pointwise=st_after_point,
        point_b0=point_batches[0], point_b1=point_batches[1],
        adj_indptr=adj.indptr.astype(np.int64), adj_indices=adj.indices.astype(np.int32),
        adj_data=adj.data.astype(np.float32), adj_shape=np.array(adj.shape),
        rmat_indptr=rmat.indptr.astype(np.int64), rmat_indices=rmat.indices.astype(np.int32),
        rmat_data=rmat.data.astype(np.float32), rmat_shape=np.array(rmat.shape),
        conf=np.array(CONF_LGCN),
    )
    print('samplers: pairwise batches', len(pair_batches), 'last', pair_batches[-1].shape,
          'pointwise b0', point_batches[0].shape, 'adj nnz', adj.nnz, 'rmat nnz', rmat.nnz)


def gen_mf():
    """One fixture per rating-prediction MF model: the order the entries were visited in each epoch
    (a permutation of the initial training list), the tables after every epoch, the epoch losses,
    the learning-rate schedule, the MT19937 state after every epoch's shuffle and the final
    MAE / RMSE lines."""
    import importlib
    from util.config import ModelConf
    from QRec import QRec
    for name, d, lr, seed in MF_RUNS:
        cname = '%s_ft.conf' % name
        with open(cname, 'w') as f:
            f.write(CONF_MF % dict(name=name, d=d, lr=lr))
        random.seed(seed)
        np.random.seed(seed)
        conf = ModelConf(cname)
        with contextlib.redirect_stdout(io.StringIO()):
            q = QRec(conf)
        cls = getattr(importlib.import_module('model.rating.' + name), name)
        model = cls(conf, q.trainingData, q.testData)
        first = list(model.data.trainingData)
        where = {id(e): k for k, e in enumerate(first)}
        rec = dict(order=[], P=[], Q=[], Bu=[], Bi=[], loss=[], lrate=[], states=[], rmse=[])
        orig_conv = cls.isConverged

        def spy_conv(self, epoch):
            rec['order'].append(np.array([where[id(e)] for e in self.data.trainingData], dtype=np.int32))
            rec['P'].append(self.P.copy())
            rec['Q'].append(self.Q.copy())
            if hasattr(self, 'Bu'):
                rec['Bu'].append(self.Bu.copy())
                rec['Bi'].append(self.Bi.copy())
            rec['loss'].append(float(self.loss))
            lr_before = self.lRate
            r = orig_conv(self, epoch)
            rec['rmse'].append([m.strip() for m in self.measure])
            rec['lrate'].append((lr_before, self.lRate))
            rec['states'].append(_state_to_array(random.getstate()))
            return r

        cls.isConverged = spy_conv
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                model.readConfiguration()
                model.initializing_log()
                state_before = _state_to_array(random.getstate())
                model.initModel()
                init = dict(P0=model.P.copy(), Q0=model.Q.copy())
                if hasattr(model, 'Bu'):
                    init.update(Bu0=model.Bu.copy(), Bi0=model.Bi.copy())
                model.trainModel()
                model.evalRatings()
        finally:
            cls.isConverged = orig_conv
        measure = [m.strip() for m in model.measure]
        print(name, 'FilmTrust: train', model.data.trainingSize(), 'losses', rec['loss'], 'measure', measure)
        extra = {}
        if rec['Bu']:
            extra = dict(Bu_last=rec['Bu'][-1], Bi_last=rec['Bi'][-1])
        np.savez_compressed(
            os.path.join(OUT, 'mf_%s_filmtrust.npz' % name.lower()),
            user_names=np.array([model.data.id2user[k] for k in range(len(model.data.user))]),
            item_names=np.array([model.data.id2item[k] for k in range(len(model.data.item))]),
            train_users=np.array([e[0] for e in first]), train_items=np.array([e[1] for e in first]),
            train_rating=np.array([e[2] for e in first], dtype=np.float64),
            test_users=np.array([e[0] for e in model.data.testData]),
            test_items=np.array([e[1] for e in model.data.testData]),
            test_rating=np.array([e[2] for e in model.data.testData], dtype=np.float64),
            test_pred=np.array([e[3] for e in model.data.testData], dtype=np.float64),
            global_mean=np.array(model.data.globalMean),
            mt_state_before=state_before, mt_state_after_epoch=np.stack(rec['states']),
            order_epoch=np.stack(rec['order']),               # [E, n] indices into the initial list
            # tables after the first epoch (fp32 copy, loose checks) and after the last (float64, exact)
            P_epoch1=rec['P'][0].astype(np.float32), Q_epoch1=rec['Q'][0].astype(np.float32),
            P_last=rec['P'][-1], Q_last=rec['Q'][-1],
            loss=np.array(rec['loss']), lrate=np.array(rec['lrate']),
            epoch_measure=np.array(rec['rmse']), measure=np.array(measure),
            seed=np.array(seed), conf=np.array(CONF_MF % dict(name=name, d=d, lr=lr)),
            **init, **extra)


CONF_SBPR = """ratings=./dataset/FilmTrust/ratings.txt
social=./dataset/FilmTrust/trust.txt
ratings.setup=-columns 0 1 2
social.setup=-columns 0 1
model.name=SBPR
evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt -b 1.0 -tf
item.ranking=on -topN 10
num.factors=16
num.max.epoch=2
batch_size=512
learnRate=-init 0.005 -max 0.1
reg.lambda=-u 0.01 -i 0.01 -b 0.01 -s 0.2
output.setup=off -dir ./results/
"""


def gen_sbpr():
    """model/ranking/SBPR.py:12-29 (PositiveSet / FPSet from FilmTrust's trust network) and :69-101 (next_batch): the
    social-feedback sets and the first minibatches of the UNMODIFIED reference class on the training split recorded in
    bpr_filmtrust_seed0.npz.  Only dicts are involved (no sets), so the stream does not depend on the hash seed."""
    from util.config import ModelConf
    from util.io import FileIO
    from model.ranking.SBPR import SBPR
    g = np.load(os.path.join(OUT, 'bpr_filmtrust_seed0.npz'), allow_pickle=True)
    train = [[u, i, float(r)] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    with open('SBPR_ft.conf', 'w') as f:
        f.write(CONF_SBPR)
    conf = ModelConf('SBPR_ft.conf')
    relation = FileIO.loadRelationship(conf, conf['social'])
    np.random.seed(0)
    random.seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = SBPR(conf, [list(r) for r in train], [], [list(r) for r in relation])
        m.readConfiguration()
        m.initModel()
    m.batch_size = 512
    users = list(m.data.user.keys())
    fp_sizes = np.array([len(m.FPSet[u]) if u in m.FPSet else 0 for u in users], dtype=np.int64)
    fp_sums = np.array([sum(m.FPSet[u].values()) if u in m.FPSet else 0 for u in users], dtype=np.int64)
    fp_first = np.array([(next(iter(m.FPSet[u])) if (u in m.FPSet and len(m.FPSet[u])) else '') for u in users])
    random.seed(77)
    batches = []
    for n, b in enumerate(m.next_batch()):
        batches.append(np.array(b, dtype=np.int64))                  # [5, batch]: u, i, k, j, S_uk
        if n == 7:
            break
    state = _state_to_array(random.getstate())
    np.savez_compressed(
        os.path.join(OUT, 'sbpr_filmtrust_seed77.npz'),
        relation_from=np.array([r[0] for r in relation]), relation_to=np.array([r[1] for r in relation]),
        relation_w=np.array([float(r[2]) for r in relation]),
        fp_sizes=fp_sizes, fp_sums=fp_sums, fp_first=fp_first,
        batches=np.stack(batches), mt_state_after_8_batches=state, conf=np.array(CONF_SBPR))
    print('sbpr: %d relations, %d users with social feedback, 8 batches of 512' % (len(relation), int((fp_sizes > 0).sum())))


def gen_reference():
    """tests/reference_cases.py run against the unmodified reference modules: the SHA-256 of each case's canonical
    result (tests/golden/reference_digests.json), and FilmTrust's ratings.txt, gzipped, as the loader cases' input."""
    import gzip
    import importlib
    import json
    import shutil
    with open(os.path.join(REF, 'dataset', 'FilmTrust', 'ratings.txt'), 'rb') as src, \
            gzip.GzipFile(os.path.join(OUT, 'filmtrust_ratings.txt.gz'), 'wb', mtime=0) as dst:
        shutil.copyfileobj(src, dst)
    sys.path.insert(0, os.path.join(REPO, 'tests'))
    import reference_cases as RC
    names = ('util.config', 'util.measure', 'util.qmath', 'util.io', 'util.dataSplit', 'data.rating', 'util.log',
             'base.recommender', 'base.iterativeRecommender', 'base.deepRecommender')
    mods = {n: importlib.import_module(n) for n in names}
    out = {}
    for name, case in sorted(RC.CASES.items()):
        work = tempfile.mkdtemp(prefix='qrec_ref_case_')
        out[name] = RC.digest(case(mods, work))
    # the SBPR class's social-feedback sets and sampler, on the data of tests/test_sbpr_cpu.py
    sys.path.insert(0, REPO)
    import test_sbpr_cpu as TS
    R = importlib.import_module('model.ranking.SBPR').SBPR
    golden_bpr = np.load(os.path.join(OUT, 'bpr_filmtrust_seed0.npz'))
    out['sbpr_sampler'] = RC.digest(TS.reference_sampler_view(R, mods['util.config'].ModelConf, golden_bpr,
                                                               tempfile.mkdtemp(prefix='qrec_ref_case_')))
    # the TBPR class under string-hash seed 0 (its joint item set is iterated in set order), in a fresh interpreter
    import test_tbpr_cpu as TT
    TT.run_with_hash_seed_0('T.reference_result(__import__("importlib").import_module("model.ranking.TBPR").TBPR, '
                            '__import__("importlib").import_module("util.config").ModelConf, golden_bpr, workdir)',
                            TT.GOLDEN_TBPR,
                            prelude='import types\nsys.modules["tensorflow"] = types.ModuleType("tensorflow")\n'
                                    'sys.modules["mkl"] = types.ModuleType("mkl")\nsys.path.append(%r)\n' % REF)
    with open(RC.DIGESTS, 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')


def main():
    what = set(sys.argv[1:]) or {'bpr', 'mf', 'sbpr', 'reference'}
    _enter_workdir()
    if 'reference' in what:
        gen_reference()
    if 'bpr' in what:
        gen_bpr()
    if 'mf' in what:
        gen_mf()
    if 'sbpr' in what:
        gen_sbpr()


if __name__ == '__main__':
    main()
