"""K15 on an H100: neighbour lists, KNN predictions and SlopeOne predictions against the float64 oracle
(oracle/knn_oracle.py) bit for bit, on FilmTrust and on seeded synthetic sets, across grid sizes, and the drop-ins
end to end against the reference's measure lines."""
import os
import sys
from collections import defaultdict

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import knn_oracle as KO   # noqa: E402

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'knn_filmtrust.npz')


def views(train, test):
    """The reference's dicts of a training and a test list of (user, item, rating)."""
    by_u, by_i, users, items = defaultdict(dict), defaultdict(dict), {}, {}
    for u, i, r in train:
        users.setdefault(u, len(users))
        items.setdefault(i, len(items))
        by_u[u][i] = r
        by_i[i][u] = r
    tu, ti = defaultdict(dict), defaultdict(dict)
    for u, i, r in test:
        tu[u][i] = r
        ti[i][u] = r
    um = {u: sum(by_u[u].values()) / len(by_u[u]) for u in users}
    im = {i: sum(by_i[i].values()) / len(by_i[i]) for i in items}
    total = sum(um.values())
    return dict(by_u=dict(by_u), by_i=dict(by_i), users=users, items=items, test_u=list(tu), test_i=list(ti), um=um,
                im=im, gm=total / len(um) if total != 0 else 0, lines=[(u, i) for u, i, _ in test])


def side(d, by):
    """(rows, row ids, column ids, query list, means) of one side."""
    if by == 'user':
        return d['by_u'], d['users'], d['items'], d['test_u'], d['um']
    return d['by_i'], d['items'], d['users'], d['test_i'], d['im']


def csr(rows, ids, col_ids):
    names = list(ids)
    rowptr = np.zeros(len(names) + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum([len(rows.get(n, {})) for n in names])
    cols = np.array([col_ids[c] for n in names for c in rows.get(n, {})], dtype=np.int32)
    vals = np.array([x for n in names for x in rows.get(n, {}).values()], dtype=np.float64)
    return rowptr, cols, vals


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_engine(d, by, sim, K, max_ctas=0):
    from qrec_b200 import engine as E
    rows, ids, col_ids, queries, means = side(d, by)
    rowptr, cols, vals = csr(rows, ids, col_ids)
    m = np.array([means[n] for n in ids], dtype=np.float64)
    metric = E.knn_metric(sim)
    sq = E.knn_squares(rowptr, vals, m, metric)
    q = np.array([ids.get(n, -1) for n in queries], dtype=np.int32)
    dev = dict(rowptr=cu(rowptr), cols=cu(cols), vals=cu(vals), means=cu(m), queries=cu(q))
    out = E.knn_neighbours(dev['rowptr'], dev['cols'], dev['vals'], cu(sq), dev['means'], len(col_ids),
                           dev['queries'], metric, K, max_ctas=max_ctas)
    return dev, out


def decode(d, by, out):
    from qrec_b200 import engine as E
    rows, ids, col_ids, queries, means = side(d, by)
    id2 = list(ids)
    ids_h, sims_h, cnt = (t.cpu().numpy() for t in out)
    res = {}
    for p, qn in enumerate(queries):
        res[qn] = [(id2[v] if v >= 0 else queries[E.KNN_COLD - v], float(s))
                   for v, s in zip(ids_h[p, :cnt[p]].tolist(), sims_h[p, :cnt[p]].tolist())]
        assert (ids_h[p, cnt[p]:] == E.KNN_PAD).all()
    return res


def check_lists(d, by, sim, K, got):
    rows, ids, col_ids, queries, means = side(d, by)
    ref = KO.sorted_lists(rows, list(ids), queries, sim, keep=K)
    for qn in queries:
        assert [n for n, _ in got[qn]] == [n for n, _ in ref[qn]], (by, sim, K, qn)
        assert np.array_equal(np.array([s for _, s in got[qn]], dtype=np.float64).view(np.uint64),
                              np.array([float(s) for _, s in ref[qn]], dtype=np.float64).view(np.uint64)), (qn,)
    return ref


@pytest.fixture(scope='module')
def ft():
    g = np.load(GOLDEN)
    train = list(zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist()))
    test = list(zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist()))
    return views(train, test)


@pytest.mark.parametrize('by', ['user', 'item'])
@pytest.mark.parametrize('sim', ['pcc', 'cos', 'euclidean'])
def test_filmtrust_lists(ft, by, sim):
    n_cand = len(side(ft, by)[1]) + len(side(ft, by)[3])
    for K in (1, 20, 100, n_cand + 5):
        _, out = run_engine(ft, by, sim, K)
        check_lists(ft, by, sim, K, decode(ft, by, out))


def synthetic(seed, n_users, n_items, n_test_users, cold_users, long_rows):
    """Zipf item popularity, ratings in half steps (ties galore), a few rows longer than a CTA, one-entry rows, users
    with no training row among the test users, and a stored rating of -1."""
    rng = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, n_items + 1) ** 1.1
    pop /= pop.sum()
    train = []
    for u in range(n_users):
        n = 1 if u % 17 == 3 else (600 if u in long_rows else int(rng.integers(2, 30)))
        for i in rng.choice(n_items, size=min(n, n_items), replace=False, p=pop):
            train.append(('u%d' % u, 'i%d' % i, float(rng.integers(1, 9)) / 2))
    train.append(('u5', 'i0', -1.0))
    test = []
    for u in list(rng.choice(n_users, n_test_users, replace=False)) + list(range(n_users, n_users + cold_users)):
        for i in rng.choice(n_items + 3, 3, replace=False):
            test.append(('u%d' % u, 'i%d' % i, 3.0))
    return views(train, test)


@pytest.fixture(scope='module')
def syn():
    return synthetic(7, 400, 700, 120, 40, {1, 2, 50})


@pytest.mark.parametrize('by', ['user', 'item'])
@pytest.mark.parametrize('sim', ['pcc', 'cos', 'euclidean'])
def test_synthetic_lists_and_grid_independence(syn, by, sim):
    K = 30
    outs = [run_engine(syn, by, sim, K, max_ctas=c)[1] for c in (0, 1, 3, 0)]
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)
    check_lists(syn, by, sim, K, decode(syn, by, outs[0]))
    # many candidates: K past every list
    big = len(side(syn, by)[1]) + len(side(syn, by)[3]) + 1
    check_lists(syn, by, sim, big, decode(syn, by, run_engine(syn, by, sim, big)[1]))


def predict(d, by, sim, K):
    from qrec_b200 import engine as E
    rows, ids, col_ids, queries, means = side(d, by)
    dev, out = run_engine(d, by, sim, K)
    qpos = {n: p for p, n in enumerate(queries)}
    if by == 'user':
        lq = [qpos[u] for u, i in d['lines']]
        lp = [col_ids.get(i, -1) for u, i in d['lines']]
    else:
        lq = [qpos[i] for u, i in d['lines']]
        lp = [col_ids.get(u, -1) for u, i in d['lines']]
    sv = E.knn_sorted_view(dev['rowptr'], dev['cols'], dev['vals'])
    pred, status = E.knn_predict(dev['rowptr'], *sv, dev['means'], d['gm'], dev['queries'],
                                 *out, cu(np.array(lq, dtype=np.int32)), cu(np.array(lp, dtype=np.int32)),
                                 by == 'user')
    return pred.cpu().numpy(), status.cpu().numpy()


def oracle_predict(d, by, sim, K):
    rows, ids, col_ids, queries, means = side(d, by)
    top = KO.sorted_lists(rows, list(ids), queries, sim, keep=max(K, 0))
    out, status = [], []
    for u, i in d['lines']:
        q, probe = (u, i) if by == 'user' else (i, u)
        try:
            out.append(float(KO.knn_predict(top, K, q, rows, probe, means.get(q), means, d['gm'], by == 'user')))
            status.append(0)
        except ZeroDivisionError:
            out.append(0.0)
            status.append(2)
    return np.array(out), np.array(status)


@pytest.mark.parametrize('by', ['user', 'item'])
@pytest.mark.parametrize('sim', ['pcc', 'cos', 'euclidean'])
@pytest.mark.parametrize('data', ['ft', 'syn'])
def test_knn_predictions(request, data, by, sim):
    d = request.getfixturevalue(data)
    for K in (0, 20):
        got, st = predict(d, by, sim, K)
        ref, rst = oracle_predict(d, by, sim, K)
        assert np.array_equal(st == 2, rst == 2)
        assert np.array_equal(got[st != 2].view(np.uint64), ref[rst != 2].view(np.uint64)), (data, by, sim, K)


def test_filmtrust_raw_predictions_equal_golden(ft):
    g = np.load(GOLDEN)
    got, st = predict(ft, 'user', 'pcc', 20)
    assert (st != 2).all() and np.array_equal(got.view(np.uint64), g['UserKNN_pcc_raw'].view(np.uint64))
    got, st = predict(ft, 'item', 'pcc', 20)
    assert (st != 2).all() and np.array_equal(got.view(np.uint64), g['ItemKNN_pcc_raw'].view(np.uint64))


def slopeone(d, max_ctas=0):
    from qrec_b200 import engine as E
    irp, icol, ival = csr(d['by_i'], d['items'], d['users'])
    urp, ucol, uval = csr(d['by_u'], d['users'], d['items'])
    im = np.array([d['im'][n] for n in d['items']])
    um = np.array([d['um'][n] for n in d['users']])
    qpos = {n: p for p, n in enumerate(d['test_i'])}
    items = np.array([d['items'].get(n, -1) for n in d['test_i']], dtype=np.int32)
    lq = np.array([qpos[i] for u, i in d['lines']], dtype=np.int32)
    lu = np.array([d['users'].get(u, -1) for u, i in d['lines']], dtype=np.int32)
    pred, status = E.slopeone_predict(cu(irp), cu(icol), cu(ival), cu(im), cu(urp), cu(ucol), cu(uval), cu(um),
                                      d['gm'], cu(items), cu(lq), cu(lu), max_ctas=max_ctas)
    return pred.cpu().numpy()


@pytest.mark.parametrize('data', ['ft', 'syn'])
def test_slopeone_predictions(request, data):
    d = request.getfixturevalue(data)
    diff, freq = KO.slopeone_tables(d['by_i'], list(d['items']), d['test_i'])
    ref = np.array([float(KO.slopeone_predict(diff, freq, d['by_u'], d['um'], d['im'], d['gm'], u, i))
                    for u, i in d['lines']])
    outs = [slopeone(d, c) for c in (0, 1, 3)]
    for o in outs:
        assert np.array_equal(o.view(np.uint64), ref.view(np.uint64))
    if data == 'ft':
        assert np.array_equal(outs[0].view(np.uint64), np.load(GOLDEN)['SlopeOne_raw'].view(np.uint64))


def test_bad_arguments_raise(ft):
    from qrec_b200 import engine as E
    dev, out = run_engine(ft, 'user', 'pcc', 5)
    sq = torch.zeros_like(dev['vals'])
    n_cols = len(ft['items'])
    args = [dev['rowptr'], dev['cols'], dev['vals'], sq, dev['means'], n_cols, dev['queries']]
    with pytest.raises(E.QRecError):
        E.knn_neighbours(*args, 3, 5)                                       # metric
    with pytest.raises(E.QRecError):
        E.knn_neighbours(*args, 0, -1)                                      # K
    with pytest.raises(E.QRecError):
        E.knn_neighbours(*args[:5], 10, args[6], 0, 5)                      # a column past n_cols
    with pytest.raises(E.QRecError):
        E.knn_neighbours(*args[:6], dev['queries'] + 10000, 0, 5)           # query out of range
    with pytest.raises(E.QRecError):
        E.knn_neighbours(*args[:6], torch.cat([dev['queries'], dev['queries'][:1]]), 0, 5)   # a row twice
    with pytest.raises(E.QRecError):
        E.knn_neighbours(args[0], args[1], args[2].float(), *args[3:], 0, 5)   # dtype
    bad_rp = args[0].clone()
    bad_rp[1] = int(bad_rp[2]) + 1
    with pytest.raises(E.QRecError):
        E.knn_neighbours(bad_rp, *args[1:], 0, 5)                           # row order
    with pytest.raises(E.QRecError):
        E.knn_predict(dev['rowptr'], *E.knn_sorted_view(dev['rowptr'], dev['cols'], dev['vals']), dev['means'], 0.0,
                      dev['queries'], *out,
                      cu(np.array([10 ** 6], dtype=np.int32)), cu(np.array([0], dtype=np.int32)), True)


CONF = """ratings=train.txt
ratings.setup=-columns 0 1 2
model.name=%(name)s
evaluation.setup=-testSet test.txt
item.ranking=off -topN 10
similarity=%(sim)s
num.neighbors=%(k)d
output.setup=on -dir ./results/
"""


def run_dropin(g, prefix, name, sim, k):
    """The drop-in on the fixture's lists (FilmTrust, or constructed case `prefix`): (measure, prediction lines)."""
    import glob
    import importlib
    import shutil
    from qrec_b200.util.config import ModelConf
    shutil.rmtree('results', ignore_errors=True)
    lists = [[list(t) for t in zip(*(g[prefix + part + '_' + c].tolist() for c in ('users', 'items', 'rating')))]
             for part in ('train', 'test')]
    cls = getattr(importlib.import_module('qrec_b200.model.rating.' + name), name)
    model = cls(ModelConf.from_string(CONF % dict(name=name, sim=sim, k=k)), *lists)
    model.execute()
    with open(glob.glob('results/*-rating-predictions*')[0]) as f:
        lines = [s.rstrip('\n') for s in f.readlines()[1:]]
    return [m.strip() for m in model.measure], lines


@pytest.mark.parametrize('tag', ['UserKNN_pcc', 'UserKNN_cos', 'UserKNN_euclidean', 'ItemKNN_pcc', 'ItemKNN_cos',
                                 'ItemKNN_euclidean', 'SlopeOne'])
def test_dropin_end_to_end(tmp_path, monkeypatch, tag):
    """The reference's prediction lines and measure lines on FilmTrust, written by the drop-in on the device."""
    g = np.load(GOLDEN)
    monkeypatch.chdir(tmp_path)
    name, _, sim = tag.partition('_')
    measure, lines = run_dropin(g, '', name, sim or 'pcc', 20)
    assert measure == g[tag + '_measure'].tolist()
    assert lines == g[tag + '_lines'].tolist()
    if tag in ('UserKNN_pcc', 'ItemKNN_pcc', 'SlopeOne'):
        assert measure == {'UserKNN_pcc': ['MAE:0.6323800801373789', 'RMSE:0.8229458971450877'],
                           'ItemKNN_pcc': ['MAE:0.7245317687464224', 'RMSE:0.9304817092341118'],
                           'SlopeOne': ['MAE:0.6220847166571261', 'RMSE:0.8356580706187597']}[tag]


def test_dropin_constructed_cases(tmp_path, monkeypatch):
    """Every recorded run on the small constructed sets (cold rows, stored -1s, a repeated line, num.neighbors -1, 0,
    2 and 50, pcc / cos / euclidean / an unknown name): the reference's lines, or its ZeroDivisionError."""
    g = np.load(GOLDEN)
    monkeypatch.chdir(tmp_path)
    errors = 0
    for n in range(len(g['case_seeds'])):
        runs = [(m, s, k, 'case%d_%s_%s_%d' % (n, m, s, k)) for m in ('UserKNN', 'ItemKNN')
                for s in g['case_sims'].tolist() for k in g['case_ks'].tolist()]
        runs.append(('SlopeOne', 'pcc', 20, 'case%d_SlopeOne' % n))
        for m, s, k, tag in runs:
            if str(g[tag + '_error']):
                with pytest.raises(ZeroDivisionError):
                    run_dropin(g, 'case%d_' % n, m, s, k)
                errors += 1
                continue
            measure, lines = run_dropin(g, 'case%d_' % n, m, s, k)
            assert measure == g[tag + '_measure'].tolist(), tag
            assert lines == g[tag + '_lines'].tolist(), tag
    assert errors > 0
