"""UserKNN, ItemKNN and SlopeOne on the CPU: the float64 oracle (oracle/knn_oracle.py) against the unmodified
reference's golden run (tests/golden/knn_filmtrust.npz), the per-pair SOURCE of the device kernels
(qrec_b200/csrc/knn_step.cuh, through tests/host_shims/knn_step_host.cpp) against the oracle, and the hazards the
fixture has to exercise for those comparisons to mean anything."""
import ctypes as C
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import knn_oracle as KO   # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'knn_filmtrust.npz')
K = 20


@pytest.fixture(scope='module')
def g():
    return dict(np.load(GOLDEN))


def lists_of(g, prefix=''):
    """(train, test) lists of (user, item, rating) of the fixture's FilmTrust run, or of constructed case `prefix`."""
    train = list(zip(*(g[prefix + 'train_' + k].tolist() for k in ('users', 'items', 'rating'))))
    test = list(zip(*(g[prefix + 'test_' + k].tolist() for k in ('users', 'items', 'rating'))))
    return train, test


def views(train, test):
    """The reference's dict views of a training and a test list: rows by user and by item, test lists, means."""
    by_u, by_i = defaultdict(dict), defaultdict(dict)
    users, items = {}, {}
    for u, i, r in train:
        users.setdefault(u, len(users))
        items.setdefault(i, len(items))
        by_u[u][i] = r
        by_i[i][u] = r
    test_u, test_i = defaultdict(dict), defaultdict(dict)
    for u, i, r in test:
        test_u[u][i] = r
        test_i[i][u] = r
    um = {u: sum(by_u[u].values()) / len(by_u[u]) for u in users}
    im = {i: sum(by_i[i].values()) / len(by_i[i]) for i in items}
    total = sum(um.values())
    gm = total / len(um) if total != 0 else 0
    return dict(by_u=dict(by_u), by_i=dict(by_i), users=list(users), items=list(items), test_u=list(test_u),
                test_i=list(test_i), um=um, im=im, gm=gm, lines=[(u, i) for u, i, _ in test])


def dataset(g):
    return views(*lists_of(g))


@pytest.fixture(scope='module')
def ds(g):
    return dataset(g)


def oracle_lists(d, model, sim):
    if model == 'UserKNN':
        return KO.sorted_lists(d['by_u'], d['users'], d['test_u'], sim)
    return KO.sorted_lists(d['by_i'], d['items'], d['test_i'], sim)


def oracle_run(d, model, sim, k):
    """The raw predictions of every test line in order, up to the first ZeroDivisionError: (raw, error name)."""
    raw = []
    if model == 'SlopeOne':
        diff, freq = KO.slopeone_tables(d['by_i'], d['items'], d['test_i'])
        predict = lambda u, i: KO.slopeone_predict(diff, freq, d['by_u'], d['um'], d['im'], d['gm'], u, i)  # noqa: E731
    elif model == 'UserKNN':
        top = oracle_lists(d, model, sim)
        predict = lambda u, i: KO.knn_predict(top, k, u, d['by_u'], i, d['um'].get(u), d['um'], d['gm'], True)  # noqa: E731
    else:
        top = oracle_lists(d, model, sim)
        predict = lambda u, i: KO.knn_predict(top, k, i, d['by_i'], u, d['im'].get(i), d['im'], d['gm'], False)  # noqa: E731
    try:
        for u, i in d['lines']:
            raw.append(float(predict(u, i)))
    except ZeroDivisionError as e:
        return raw, type(e).__name__
    return raw, ''


@pytest.fixture(scope='module')
def lists(ds):
    return {(m, s): oracle_lists(ds, m, s) for m in ('UserKNN', 'ItemKNN') for s in ('pcc', 'cos', 'euclidean')}


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize('sim', ['pcc', 'cos', 'euclidean'])
@pytest.mark.parametrize('model', ['UserKNN', 'ItemKNN'])
def test_oracle_lists_match_golden(g, lists, model, sim):
    tag = '%s_%s' % (model, sim)
    top = lists[(model, sim)]
    queries = g[tag + '_queries'].tolist()
    assert list(top) == queries
    keep = g[tag + '_top_names'].shape[1]
    assert keep == (32 if sim == 'pcc' else K)
    for p, q in enumerate(queries):
        n = min(keep, len(top[q]))
        assert len(top[q]) == g[tag + '_top_len'][p]
        assert [name for name, _ in top[q][:n]] == g[tag + '_top_names'][p][:n].tolist(), (tag, q)
        assert np.array_equal(bits([s for _, s in top[q][:n]]), bits(g[tag + '_top_sims'][p][:n])), (tag, q)
    if sim == 'pcc':
        chosen = [k for k in ('first', 'last', 'tie', 'cold') if '%s_full_%s_query' % (tag, k) in g]
        assert {'first', 'last', 'tie'} <= set(chosen)
        for key in chosen:
            q = str(g['%s_full_%s_query' % (tag, key)])
            assert [name for name, _ in top[q]] == g['%s_full_%s_names' % (tag, key)].tolist(), (tag, key)
            assert np.array_equal(bits([s for _, s in top[q]]), bits(g['%s_full_%s_sims' % (tag, key)])), (tag, key)


@pytest.mark.parametrize('tag', ['UserKNN_pcc', 'UserKNN_cos', 'UserKNN_euclidean', 'ItemKNN_pcc', 'ItemKNN_cos',
                                 'ItemKNN_euclidean', 'SlopeOne'])
def test_oracle_predictions_match_golden(g, ds, tag):
    model, _, sim = tag.partition('_')
    raw, error = oracle_run(ds, model, sim or 'pcc', K)
    assert not error and np.array_equal(bits(raw), bits(g[tag + '_raw']))


def case_runs(g):
    """(case prefix, model, similarity, k, fixture tag) of every recorded constructed run."""
    out = []
    for n in range(len(g['case_seeds'])):
        for m in ('UserKNN', 'ItemKNN'):
            for s in g['case_sims'].tolist():
                for k in g['case_ks'].tolist():
                    out.append(('case%d_' % n, m, s, k, 'case%d_%s_%s_%d' % (n, m, s, k)))
        out.append(('case%d_' % n, 'SlopeOne', 'pcc', K, 'case%d_SlopeOne' % n))
    return out


def test_oracle_matches_constructed_cases(g):
    errors = 0
    for prefix, m, s, k, tag in case_runs(g):
        d = views(*lists_of(g, prefix))
        raw, error = oracle_run(d, m, s, k)
        assert error == str(g[tag + '_error']), tag
        assert np.array_equal(bits(raw), bits(g[tag + '_raw'])), tag
        errors += bool(error)
    assert errors > 0                     # the reference's ZeroDivisionError is among them


def test_constructed_cases_cover_the_edges(g):
    for n in range(len(g['case_seeds'])):
        train, test = lists_of(g, 'case%d_' % n)
        pairs = [(u, i) for u, i, _ in train]
        assert len(set(pairs)) < len(pairs)                              # a repeated training line
        assert any(r == -1.0 for _, _, r in train)                       # a stored -1
        users, items = {u for u, _, _ in train}, {i for _, i, _ in train}
        assert any(u not in users for u, _, _ in test) and any(i not in items for _, i, _ in test)
    assert 'foo' in g['case_sims'].tolist() and {0, 50} <= set(g['case_ks'].tolist()) and min(g['case_ks']) < 0


def test_measure_lines(g):
    assert list(g['UserKNN_pcc_measure']) == ['MAE:0.6323800801373789', 'RMSE:0.8229458971450877']
    assert list(g['ItemKNN_pcc_measure']) == ['MAE:0.7245317687464224', 'RMSE:0.9304817092341118']
    assert list(g['SlopeOne_measure']) == ['MAE:0.6220847166571261', 'RMSE:0.8356580706187597']


def test_fixture_exercises_the_hazards(g, ds):
    # ties across the K boundary decide the neighbour set
    for model in ('UserKNN', 'ItemKNN'):
        sims, n = g[model + '_pcc_top_sims'], g[model + '_pcc_top_len']
        tied = int(((n > K) & (sims[:, K - 1] == sims[:, K])).sum())
        assert tied > len(n) // 2, (model, tied)
    # a pair's bits depend on which row is x1
    pairs = [(a, b) for a in ds['test_u'][:40] if a in ds['by_u'] for b in ds['users'][:200] if b != a]
    asym = sum(KO.similarity(ds['by_u'][a], ds['by_u'][b], 'pcc') != KO.similarity(ds['by_u'][b], ds['by_u'][a], 'pcc')
               for a, b in pairs)
    assert asym > 0
    # CPython's ** 2 differs from numpy's square on some of the centred ratings
    cen = [x - ds['um'][u] for u, row in ds['by_u'].items() for x in row.values()]
    pw = np.array([c ** 2 for c in cen])
    assert int((bits(pw) != bits(np.square(np.array(cen)))).sum()) > 0


@pytest.fixture(scope='module')
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libknn_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'knn_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    dp, i32p, i64p = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    lib.host_knn_similarity.restype = None
    lib.host_knn_similarity.argtypes = [C.c_int32, i64p, i32p, dp, dp, dp, C.c_int32, i32p, i32p, C.c_int64, dp]
    return lib


def squares(vals, means, sim):
    """engine.knn_squares restated: CPython's ** 2 per entry."""
    if sim == 'pcc':
        return np.array([(x - m) ** 2 for x, m in zip(vals, means)])
    return np.array([x ** 2 for x in vals])


@pytest.mark.parametrize('sim,metric', [('pcc', 0), ('cos', 1), ('euclidean', 2)])
def test_header_shim_matches_oracle(ds, shim, sim, metric):
    names = ds['users']
    rows = [ds['by_u'][u] for u in names]
    col_of = {i: k for k, i in enumerate(ds['items'])}
    rowptr = np.zeros(len(rows) + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    cols = np.array([col_of[i] for r in rows for i in r], dtype=np.int32)
    vals = np.array([x for r in rows for x in r.values()], dtype=np.float64)
    means = np.array([ds['um'][u] for u in names], dtype=np.float64)
    sq = squares(vals.tolist(), np.repeat(means, np.diff(rowptr)).tolist(), sim)
    rng = np.random.default_rng(3)
    x1 = rng.integers(0, len(names), 4000).astype(np.int32)
    x2 = rng.integers(0, len(names), 4000).astype(np.int32)
    out = np.empty(len(x1))
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))   # noqa: E731
    shim.host_knn_similarity(metric, P(rowptr, C.c_int64), P(cols, C.c_int32), P(vals, C.c_double),
                             P(np.ascontiguousarray(sq), C.c_double), P(means, C.c_double), len(col_of),
                             P(x1, C.c_int32), P(x2, C.c_int32), len(x1), P(out, C.c_double))
    ref = [float(KO.similarity(rows[a], rows[b], sim)) for a, b in zip(x1.tolist(), x2.tolist())]
    assert np.array_equal(bits(out), bits(ref))


# ---------------------------------------------------------------------------------------------------------------------
# the drop-ins' life cycle, with the oracle in place of the K15 launches (CPU tensors)
# ---------------------------------------------------------------------------------------------------------------------
def _rows(rowptr, cols, vals):
    rp, cl, vl = rowptr.numpy(), cols.numpy(), vals.numpy()
    return {r: dict(zip(cl[rp[r]:rp[r + 1]].tolist(), vl[rp[r]:rp[r + 1]].tolist())) for r in range(len(rp) - 1)}


class OracleEngine(object):
    """engine.knn_neighbours / knn_sorted_view / knn_predict / slopeone_predict restated with oracle/knn_oracle.py
    on CPU tensors, with the engine's conventions (cold earlier queries as KNN_COLD - position, padding, status 2
    for the reference's ZeroDivisionError).  Counts the lines of every predict call."""

    def __init__(self, E):
        self.E = E
        self.batches = []

    def knn_neighbours(self, rowptr, cols, vals, sq, means, n_cols, queries, metric, K, max_ctas=0):
        import torch
        rows = _rows(rowptr, cols, vals)
        names = [q if q >= 0 else ('cold', p) for p, q in enumerate(queries.tolist())]
        top = KO.sorted_lists(rows, list(rows), names, self.E.KNN_METRICS[metric], keep=K)
        ids = torch.full((len(names), K), self.E.KNN_PAD, dtype=torch.int32)
        sims = torch.zeros((len(names), K), dtype=torch.float64)
        cnt = torch.zeros(len(names), dtype=torch.int32)
        for p, q in enumerate(names):
            cnt[p] = len(top[q])
            for k, (n, s) in enumerate(top[q]):
                ids[p, k] = n if not isinstance(n, tuple) else self.E.KNN_COLD - n[1]
                sims[p, k] = float(s)
        return ids, sims, cnt

    def knn_sorted_view(self, rowptr, cols, vals):
        return cols, vals          # knn_predict below reads the rows as dicts

    def knn_predict(self, rowptr, scols, svals, means, global_mean, queries, ids, sims, counts, line_qpos, line_probe,
                    minus_one_unrated):
        import torch
        rows = _rows(rowptr, scols, svals)
        m = dict(enumerate(means.tolist()))
        q = queries.tolist()
        pred, status = [], []
        self.batches.append(line_qpos.shape[0])
        for p, x in zip(line_qpos.tolist(), line_probe.tolist()):
            top = {p: [(int(n), float(s)) for n, s in zip(ids[p, :counts[p]].tolist(), sims[p, :counts[p]].tolist())]}
            try:
                pred.append(float(KO.knn_predict(top, ids.shape[1], p, rows, x, m[q[p]] if q[p] >= 0 else None, m,
                                                 global_mean, minus_one_unrated)))
                status.append(0)
            except ZeroDivisionError:
                pred.append(0.0)
                status.append(2)
        return torch.tensor(pred, dtype=torch.float64), torch.tensor(status, dtype=torch.int32)

    def slopeone_predict(self, irp, icols, ivals, imeans, urp, ucols, uvals, umeans, global_mean, test_items,
                         line_qpos, line_user, max_ctas=0):
        import torch
        items, users = _rows(irp, icols, ivals), _rows(urp, ucols, uvals)
        names = [i if i >= 0 else ('cold', p) for p, i in enumerate(test_items.tolist())]
        diff, freq = KO.slopeone_tables(items, list(items), names)
        um, im = dict(enumerate(umeans.tolist())), dict(enumerate(imeans.tolist()))
        self.batches.append(line_qpos.shape[0])
        pred = [float(KO.slopeone_predict(diff, freq, users, um, im, global_mean, u if u >= 0 else ('cold', -1),
                                          names[p]))
                for p, u in zip(line_qpos.tolist(), line_user.tolist())]
        return torch.tensor(pred, dtype=torch.float64), torch.zeros(len(pred), dtype=torch.int32)


@pytest.fixture
def oracle_engine(monkeypatch, tmp_path):
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.model.rating._knn import KNNRating
    from qrec_b200.model.rating.SlopeOne import SlopeOne
    fake = OracleEngine(E)
    for name in ('knn_neighbours', 'knn_sorted_view', 'knn_predict', 'slopeone_predict'):
        monkeypatch.setattr(E, name, getattr(fake, name))
    for cls in (KNNRating, SlopeOne):
        monkeypatch.setattr(cls, '_device', lambda self: torch.device('cpu'))
    monkeypatch.chdir(tmp_path)
    return fake


CONF = """ratings=train.txt
ratings.setup=-columns 0 1 2
model.name=%(name)s
evaluation.setup=-testSet test.txt
item.ranking=%(ranking)s -topN 10
similarity=%(sim)s
num.neighbors=%(k)d
output.setup=on -dir ./results/
"""


def dropin(name, sim, k, train, test, ranking='off'):
    import importlib
    from qrec_b200.util.config import ModelConf
    conf = ModelConf.from_string(CONF % dict(name=name, sim=sim, k=k, ranking=ranking))
    cls = getattr(importlib.import_module('qrec_b200.model.rating.' + name), name)
    return cls(conf, [list(t) for t in train], [list(t) for t in test])


def written_lines():
    import glob
    with open(glob.glob('results/*-rating-predictions*')[0]) as f:
        return [s.rstrip('\n') for s in f.readlines()[1:]]


@pytest.mark.parametrize('tag', ['UserKNN_pcc', 'ItemKNN_cos', 'ItemKNN_euclidean', 'SlopeOne'])
def test_dropin_life_cycle_filmtrust(g, oracle_engine, tag, capsys):
    name, _, sim = tag.partition('_')
    model = dropin(name, sim or 'pcc', K, *lists_of(g))
    model.execute()
    out = capsys.readouterr().out
    assert [m.strip() for m in model.measure] == g[tag + '_measure'].tolist()
    assert written_lines() == g[tag + '_lines'].tolist()
    if name == 'SlopeOne':
        assert out.count(' finished.\n') == len(model.data.testSet_i)
        return
    noun = 'user' if name == 'UserKNN' else 'item'
    assert 'Computing %s similarities...' % noun in out and 'The %s similarities have been calculated.' % noun in out
    assert out.count('progress:') == (len(g[tag + '_queries']) + 99) // 100
    top = model.topUsers if name == 'UserKNN' else model.topItems
    assert list(top) == g[tag + '_queries'].tolist()
    keep = g[tag + '_top_names'].shape[1]
    for p, q in enumerate(top):
        n = min(K, g[tag + '_top_len'][p])
        assert len(top[q]) == n
        assert [a for a, _ in top[q]] == g[tag + '_top_names'][p][:min(n, keep)].tolist()
        assert np.array_equal(bits([s for _, s in top[q]]), bits(g[tag + '_top_sims'][p][:n]))
    # a pair outside the test list goes through the same path as a one-line batch
    q = next(iter(top))
    other = next(c for c in (model.data.item if name == 'UserKNN' else model.data.user)
                 if (q, c) not in model._pred and (c, q) not in model._pred)
    pair = (q, other) if name == 'UserKNN' else (other, q)
    before = len(oracle_engine.batches)
    got = model.predictForRating(*pair)
    assert oracle_engine.batches[before:] == [1]
    d = views(*lists_of(g))
    lst = oracle_lists(d, name, sim)
    ref = (KO.knn_predict(lst, K, q, d['by_u'], other, d['um'].get(q), d['um'], d['gm'], True) if name == 'UserKNN'
           else KO.knn_predict(lst, K, q, d['by_i'], other, d['im'].get(q), d['im'], d['gm'], False))
    assert bits(got) == bits(ref)


def test_dropin_life_cycle_constructed_cases(g, oracle_engine, capsys):
    """Cold users and items, cold earlier queries in the neighbour lists, stored -1s, num.neighbors <= 0 and past the
    lists, an unknown similarity name, and the reference's ZeroDivisionError: every recorded run through the drop-in."""
    import shutil
    cold_neighbours = 0
    for prefix, m, s, k, tag in case_runs(g):
        shutil.rmtree('results', ignore_errors=True)
        model = dropin(m, s, k, *lists_of(g, prefix))
        if str(g[tag + '_error']):
            with pytest.raises(ZeroDivisionError):
                model.execute()
            continue
        model.execute()
        assert [x.strip() for x in model.measure] == g[tag + '_measure'].tolist(), tag
        assert written_lines() == g[tag + '_lines'].tolist(), tag
        top = getattr(model, 'topUsers', None) or getattr(model, 'topItems', None) or {}
        known = model.data.user if m == 'UserKNN' else model.data.item
        cold_neighbours += sum(n not in known for row in top.values() for n, _ in row)
        if m != 'SlopeOne':
            assert all(len(row) == (0 if k <= 0 else min(k, len(row))) for row in top.values())
    capsys.readouterr()
    assert cold_neighbours > 0           # a cold earlier query was decoded into the lists


def test_dropin_ranking_exits(g, oracle_engine, capsys):
    for name in ('UserKNN', 'ItemKNN'):
        model = dropin(name, 'pcc', K, *lists_of(g, 'case0_'), ranking='on')
        with pytest.raises(SystemExit) as e:
            model.execute()
        assert e.value.code == 0
        assert ('So ranking for all items in %s is not available.' % name) in capsys.readouterr().out
