"""Cases that compare this project's Python drop-in surface with the unmodified reference modules.

Each case takes a dict of modules under the reference's own names ('util.config', 'base.recommender', ...) and a
scratch directory, and returns what the comparison looks at.  oracle/gen_golden.py runs every case once against the
reference and stores the SHA-256 of its canonical form in tests/golden/reference_digests.json; the tests run the
same case against qrec_b200 and require the same digest, i.e. exactly equal results.  The inputs are seeded, and
the FilmTrust ratings file the loader cases read is stored gzipped under tests/golden/.
"""
import contextlib
import gzip
import hashlib
import io
import json
import os
import random
import shutil

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
DIGESTS = os.path.join(GOLDEN, 'reference_digests.json')
RATINGS_GZ = os.path.join(GOLDEN, 'filmtrust_ratings.txt.gz')


def canonical(x):
    """A JSON-able form in which equal results are equal: dict items sorted by key, sequences as lists, arrays as
    lists, floats by repr (exact)."""
    if isinstance(x, dict):
        return ['dict', sorted(([canonical(k), canonical(v)] for k, v in x.items()), key=lambda kv: json.dumps(kv[0]))]
    if isinstance(x, np.ndarray):
        return canonical(x.tolist())
    if isinstance(x, (list, tuple)):
        return [canonical(v) for v in x]
    if isinstance(x, (bool, np.bool_)):
        return bool(x)
    if isinstance(x, (int, np.integer)):
        return int(x)
    if isinstance(x, (float, np.floating)):
        return 'f' + repr(float(x))
    if x is None or isinstance(x, str):
        return x
    raise TypeError('no canonical form for %r' % type(x))


def digest(x):
    return hashlib.sha256(json.dumps(canonical(x), separators=(',', ':')).encode()).hexdigest()


def ratings_file(workdir):
    """FilmTrust's ratings.txt (as shipped with the reference) unpacked into workdir."""
    path = os.path.join(workdir, 'ratings.txt')
    if not os.path.exists(path):
        with gzip.open(RATINGS_GZ, 'rb') as src, open(path, 'wb') as dst:
            shutil.copyfileobj(src, dst)
    return path


def _conf(mods, mapping):
    c = mods['util.config'].ModelConf.__new__(mods['util.config'].ModelConf)
    c.config = dict(mapping)
    return c


def _parse(text):
    return dict(line.split('=', 1) for line in text.splitlines() if line.strip())


def case_option_conf(mods, workdir):
    R = mods['util.config'].OptionConf
    rng = random.Random(0)
    vocab = ['on', 'off', '-a', '-b', '--c', '-topN', '-1', '-12', '-0.5', '5', '10,20', 'x', '0.1', '-tf', '', '-n_layer', '2']
    out = []
    for _ in range(3000):
        s = ' '.join(rng.choice(vocab) for _ in range(rng.randint(1, 8)))
        if rng.random() < 0.2:
            s = ' ' + s + ' '
        o = R(s)
        out.append([s, o.options, o.isMainOn(), o.line])
    return out


def case_model_conf(mods, workdir):
    """Seeded configuration files in the shapes QRec's config/*.conf use (key=value, option strings, blank lines,
    malformed lines), and the malformed file of the original test."""
    rng = random.Random(4)
    keys = ['ratings', 'ratings.setup', 'model.name', 'evaluation.setup', 'item.ranking', 'num.factors', 'num.max.epoch',
            'learnRate', 'reg.lambda', 'output.setup', 'social', 'social.setup', 'batch_size', 'SGL', 'SimGCL']
    vals = ['./dataset/FilmTrust/trainset.txt', '-columns 0 1 2', 'BPR', '-testSet ./dataset/FilmTrust/testset.txt',
            'on -topN 10,20', '64', '30', '-init 0.01 -max 1', '-u 0.001 -i 0.001 -b 0.2 -s 0.2', 'on -dir ./results/',
            '-n_layer 2 -lambda 0.01 -droprate 0.1 -augtype 1 -temp 0.2', 'x y', '']
    out = []
    for k in range(40):
        lines = []
        for _ in range(rng.randint(1, 14)):
            r = rng.random()
            if r < 0.75:
                lines.append('%s=%s' % (rng.choice(keys), rng.choice(vals)))
            elif r < 0.85:
                lines.append('')
            elif r < 0.93:
                lines.append('not a pair')
            else:
                lines.append('a=b=c')
        path = os.path.join(workdir, 'conf%d.conf' % k)
        with open(path, 'w') as f:
            f.write('\n'.join(lines) + '\n')
        with contextlib.redirect_stdout(io.StringIO()):
            out.append(mods['util.config'].ModelConf(path).config)
    bad = os.path.join(workdir, 'bad.conf')
    with open(bad, 'w') as f:
        f.write('a=1\nnot a pair\nb=2=3\n\nc=x y\n')
    with contextlib.redirect_stdout(io.StringIO()):
        out.append(mods['util.config'].ModelConf(bad).config)
    return out


def case_measures(mods, workdir):
    R = mods['util.measure'].Measure
    rng = random.Random(1)
    items = ['i%d' % k for k in range(60)]
    out = []
    for _ in range(200):
        users = ['u%d' % k for k in range(rng.randint(1, 12))]
        origin = {u: {it: 1.0 for it in rng.sample(items, rng.randint(1, 15))} for u in users}
        res = {u: [(it, rng.random()) for it in rng.sample(items, 20)] for u in users}
        tops = sorted(rng.sample([1, 3, 5, 10, 20], rng.randint(1, 3)))
        out.append(R.rankingMeasure(origin, res, tops))
    rows = [['u', 'i', rng.random() * 5, rng.random() * 5] for _ in range(50)]
    out.append(R.ratingMeasure(rows))
    out.append(R.ratingMeasure([]))
    return out


def case_find_k_largest(mods, workdir):
    F = mods['util.qmath'].find_k_largest
    rng = np.random.default_rng(2)
    out = []
    for trial in range(120):
        n, K = int(rng.integers(3, 300)), int(rng.integers(1, 15))
        s = rng.standard_normal(n).round(1 if trial % 3 == 0 else 7)
        s[rng.integers(0, n, n // 5)] = 0.0                       # rated items are overwritten with 0
        ids, vals = F(K, s.copy())
        out.append([list(ids), list(vals)])
    out.append(mods['util.qmath'].sigmoid(0.3))
    return out


def case_rating(mods, workdir):
    RR = mods['data.rating'].Rating
    rng = random.Random(3)
    out = []
    for ev in ('-ap 0.2', '-ap 0.2 -b 1', '-cold 2', '-val 0.25'):
        train = [['u%d' % rng.randint(0, 30), 'i%d' % rng.randint(0, 40), float(rng.randint(1, 5))] for _ in range(400)]
        test = [['u%d' % rng.randint(0, 35), 'i%d' % rng.randint(0, 45), float(rng.randint(1, 5))] for _ in range(120)]
        random.seed(11)
        r = RR(_conf(mods, {'ratings': 'x', 'evaluation.setup': ev}), [x[:] for x in train], [x[:] for x in test])
        got = {a: getattr(r, a) for a in ('user', 'item', 'id2user', 'id2item', 'userMeans', 'itemMeans', 'globalMean',
                                          'rScale', 'trainingData', 'testData')}
        got['sets'] = [dict(r.trainSet_u), dict(r.testSet_u), dict(r.trainSet_i), dict(r.testSet_i)]
        got['sizes'] = [r.trainingSize(), r.testSize()]
        u0 = next(iter(r.user))
        got['u0'] = [r.userRated(u0), r.row(u0)]
        out.append([ev, got])
    return out


def case_data_split(mods, workdir):
    RS = mods['util.dataSplit'].DataSplit
    rng = random.Random(5)
    data = [['u%d' % rng.randint(0, 9), 'i%d' % rng.randint(0, 9), float(rng.randint(0, 1))] for _ in range(300)]
    out = []
    for ratio, binar in ((0.2, False), (0.2, True), (1.5, False), (0.0, True)):
        random.seed(7)
        out.append([RS.dataSplit(data, test_ratio=ratio, binarized=binar), random.getstate()])
    for k, binar in ((5, False), (3, True), (1, False), (11, False)):
        out.append(list(RS.crossValidation(data, k, binarized=binar)))
    return out


def case_loader(mods, workdir):
    RF = mods['util.io'].FileIO
    path = ratings_file(workdir)
    out = []
    for setup, kw in (('-columns 0 1 2', {}), ('-columns 0 1 2', {'binarized': True, 'threshold': 3.0}),
                      ('-columns 1 0', {}), ('-columns 0 1 2 -header', {'bTest': True})):
        with contextlib.redirect_stdout(io.StringIO()):
            out.append(RF.loadDataSet(_conf(mods, {'ratings.setup': setup}), path, **kw))
    return out


def case_eval_ranking(mods, workdir):
    """Recommender.evalRanking / IterativeRecommender.isConverged fed the same numpy P, Q: recommendation lines,
    metric strings, learning-rate updates and generator state."""
    Cls = mods['base.iterativeRecommender'].IterativeRecommender
    rng = random.Random(9)
    conf_text = ('ratings=x\nratings.setup=-columns 0 1 2\nmodel.name=BPR\nevaluation.setup=-ap 0.2 -b 1\n'
                 'item.ranking=on -topN 5,10\nnum.factors=8\nnum.max.epoch=3\nlearnRate=-init 0.01 -max 0.0105\n'
                 'reg.lambda=-u 0.001 -i 0.001 -b 0.2 -s 0.2\noutput.setup=on -dir ./results/\n')
    train = [['u%d' % rng.randint(0, 40), 'i%d' % rng.randint(0, 60), 1.0] for _ in range(900)]
    test = [['u%d' % rng.randint(0, 45), 'i%d' % rng.randint(0, 60), 1.0] for _ in range(200)]
    cwd = os.getcwd()
    os.chdir(workdir)
    try:
        m = Cls(_conf(mods, _parse(conf_text)), [r[:] for r in train], [r[:] for r in test])
        with contextlib.redirect_stdout(io.StringIO()):
            m.readConfiguration()
            m.initializing_log()
            np.random.seed(4)
            m.initModel()
            random.seed(21)
            conv = []
            for epoch, loss in enumerate([100.0, 90.0, 95.0, 94.9995], 1):
                m.loss = loss
                conv.append((m.isConverged(epoch), m.lRate))
            m.evalRanking()
    finally:
        os.chdir(cwd)
    return [conv, m.recOutput, m.measure, random.getstate(), [r[:] for r in m.data.trainingData]]


def case_minibatch_samplers(seed):
    def case(mods, workdir):
        Cls = mods['base.deepRecommender'].DeepRecommender
        rng = random.Random(seed)
        conf_text = ('ratings=x\nratings.setup=-columns 0 1 2\nmodel.name=LightGCN\nevaluation.setup=-ap 0.2\n'
                     'item.ranking=on -topN 10\nnum.factors=8\nnum.max.epoch=1\nbatch_size=128\n'
                     'learnRate=-init 0.01 -max 1\nreg.lambda=-u 0.001 -i 0.001 -b 0.2 -s 0.2\noutput.setup=off -dir ./results/\n')
        train = [['u%d' % rng.randint(0, 50), 'i%d' % rng.randint(0, 80), float(rng.randint(1, 5))] for _ in range(1000)]
        cwd = os.getcwd()
        os.chdir(workdir)
        try:
            m = Cls(_conf(mods, _parse(conf_text)), [r[:] for r in train], [])
            with contextlib.redirect_stdout(io.StringIO()):
                m.readConfiguration()
            random.seed(seed)
            pair = [[np.asarray(x).tolist() for x in batch] for batch in m.next_batch_pairwise()]
            point = [[np.asarray(x).tolist() for x in batch] for batch in m.next_batch_pointwise()]
        finally:
            os.chdir(cwd)
        return [pair, point, [r[:] for r in m.data.trainingData], random.getstate()]
    return case


def case_interaction_table_ids(mods, workdir):
    """The reference's id space for the FilmTrust file: loader + Rating (the array-backed table must reproduce it)."""
    path = ratings_file(workdir)
    rc = _conf(mods, {'ratings.setup': '-columns 0 1 2', 'evaluation.setup': '-ap 0.2 -b 1'})
    with contextlib.redirect_stdout(io.StringIO()):
        recs = mods['util.io'].FileIO.loadDataSet(rc, path, binarized=True, threshold=1.0)
    data = mods['data.rating'].Rating(rc, recs, [])
    return [len(recs), [data.id2user[k] for k in range(len(data.user))], [data.id2item[k] for k in range(len(data.item))],
            [data.user[r[0]] for r in recs], [data.item[r[1]] for r in recs]]


CASES = {
    'option_conf': case_option_conf,
    'model_conf': case_model_conf,
    'measures': case_measures,
    'find_k_largest': case_find_k_largest,
    'rating': case_rating,
    'data_split': case_data_split,
    'loader': case_loader,
    'eval_ranking': case_eval_ranking,
    'minibatch_samplers_0': case_minibatch_samplers(0),
    'minibatch_samplers_7': case_minibatch_samplers(7),
    'minibatch_samplers_2024': case_minibatch_samplers(2024),
    'interaction_table_ids': case_interaction_table_ids,
}


def qrec_b200_modules():
    """This project's modules under the reference's names."""
    import importlib
    names = ('util.config', 'util.measure', 'util.qmath', 'util.io', 'util.dataSplit', 'data.rating', 'util.log',
             'base.recommender', 'base.iterativeRecommender', 'base.deepRecommender')
    return {n: importlib.import_module('qrec_b200.' + n) for n in names}


def recorded(name):
    with open(DIGESTS) as f:
        return json.load(f)[name]
