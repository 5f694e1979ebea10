"""EE and SREE without a GPU: the numpy oracle against the reference's golden runs, the device step source compiled on
the host, and the engine wrappers' input checks."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import ee_sree_oracle as EO             # noqa: E402
from oracle import socialmf_soreg_oracle as SM      # noqa: E402
from oracle import sorec_rste_oracle as SR          # noqa: E402
from test_social_rating_cpu import _d, conf_value, orders   # noqa: E402
from test_socialmf_soreg_cpu import _csr            # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
TAGS = ['ee', 'sree_w', 'sree_nw']
LISTS = ('user_names', 'item_names', 'train_users', 'train_items', 'train_rating', 'test_users', 'test_items',
         'test_rating')


def film(name):
    """A FilmTrust run; the SREE file shares the id maps and lists of the EE one."""
    g = dict(np.load(os.path.join(GOLD, '%s_filmtrust.npz' % name.lower())))
    if name == 'SREE':
        ee = np.load(os.path.join(GOLD, 'ee_filmtrust.npz'))
        g.update({k: ee[k] for k in LISTS})
    return g


def cases():
    z = np.load(os.path.join(GOLD, 'ee_sree_cases.npz'))
    return {tag: {k.split('/', 1)[1]: z[k] for k in z.files if k.startswith(tag + '/')} for tag in z['tags'].tolist()}


def case_files():
    z = np.load(os.path.join(GOLD, 'ee_sree_cases.npz'))
    return {k.split('/', 1)[1]: z[k] for k in z.files if k.startswith('files/')}


def model_of(g):
    return 'SREE' if 'raw_u1' in g else 'EE'


def load_run(g):
    """ids and the id-mapped training list of a run, in file order."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    u0 = np.array([users[x] for x in g['train_users'].tolist()], np.int32)
    i0 = np.array([items[x] for x in g['train_items'].tolist()], np.int32)
    return users, items, u0, i0


def social_of(g):
    """(visit, followee lists by id, followers by id, followees by name) of a SREE run, from the relation list as
    read."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    names = g['user_names'].tolist()
    raw = list(zip(g['raw_u1'].tolist(), g['raw_u2'].tolist(), g['raw_w'].tolist()))
    followees, followers, _ = SR.clean_social(users, raw)
    first = []
    for a, b, _ in raw:
        for x in (a, b):
            if x not in first:
                first.append(x)
    assert first == g['social_user'].tolist()
    visit = SM.visit_ids(first, users)
    return (visit, SM.neighbour_lists(names, users, followees), SM.neighbour_lists(names, users, followers),
            followees)


def hyper(g):
    return dict(reg_u=conf_value(g, 'reg.lambda', '-u'), reg_i=conf_value(g, 'reg.lambda', '-i'),
                reg_b=conf_value(g, 'reg.lambda', '-b'), global_mean=float(g['global_mean']))


def initial(g, dtype=np.float64):
    users, items, _, _ = load_run(g)
    U, I, d = len(users), len(items), _d(g)
    P, Q = SR.initial_tables(int(g['seed']), U, I, d, False)
    Bu, Bi = EO.initial_biases(int(g['seed']), U, I, d)
    return [t.astype(dtype) for t in (P, Q, Bu, Bi)]


def replay(g, dtype=np.float64):
    """The oracle over the recorded visiting orders: (tables after epoch 1, after the last epoch, losses, rates)."""
    _, _, u0, i0 = load_run(g)
    tables = initial(g, dtype)
    h = hyper(g)
    social = model_of(g) == 'SREE'
    if social:
        visit, fl, _, _ = social_of(g)
    lr, last = float(g['lrate'][0][0]), 0.0
    losses, lrs, first = [], [], None
    for e, o in enumerate(orders(g)):
        args = (*tables, u0[o], i0[o], g['train_rating'][o])
        if social:
            loss = EO.sree_epoch(*args, visit, fl, lr, h['reg_u'], h['reg_i'], h['reg_b'], h['global_mean'],
                                 conf_value(g, 'SREE', '-alpha'))
        else:
            loss = EO.ee_epoch(*args, lr, h['reg_u'], h['reg_i'], h['reg_b'], h['global_mean'])
        losses.append(loss)
        before = lr
        if not abs(last - loss) < 1e-3:
            lr = SR.update_learning_rate(lr, 1.0, e + 1, last, loss)
        lrs.append((before, lr))
        last = loss
        if e == 0:
            first = [t.copy() for t in tables]
    return first, tables, losses, lrs


def predictions(g, P, Q, Bu, Bi):
    """Each test line's prediction (globalMean for an unknown user or item), clipped as checkRatingBoundary does; and
    the measure lines of that list."""
    from qrec_b200.util.measure import Measure
    users, items, _, _ = load_run(g)
    gm = float(g['global_mean'])
    lo, hi = min(g['train_rating']), max(g['train_rating'])
    res = []
    for un, it, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist()):
        pred = (EO.predict(P, Q, Bu, Bi, users[un], items[it], gm) if un in users and it in items else gm)
        res.append([un, it, r, hi if pred > hi else lo if pred < lo else round(pred, 3)])
    return [x[3] for x in res], [m.strip() for m in Measure.ratingMeasure(res)]


def _check(g):
    first, tables, losses, lrs = replay(g)
    for t, k in zip(tables, ('P', 'Q', 'Bu', 'Bi')):
        assert np.array_equal(t, g[k + '_last']), k
    for t, k in zip(first, ('P', 'Q', 'Bu', 'Bi')):
        assert np.array_equal(t.astype(np.float32), g[k + '_epoch1']), k
    assert losses == g['loss'].tolist()
    assert np.array_equal(np.array(lrs), g['lrate'])
    preds, measure = predictions(g, *tables)
    assert preds == g['test_pred'].tolist()
    assert measure == g['measure'].tolist()


@pytest.mark.parametrize('name', ['EE', 'SREE'])
def test_oracle_reproduces_the_filmtrust_run_bit_for_bit(name):
    _check(film(name))


@pytest.mark.parametrize('tag', TAGS)
def test_oracle_reproduces_the_constructed_runs_bit_for_bit(tag):
    _check(cases()[tag])


@pytest.mark.parametrize('source', ['EE', 'SREE'] + TAGS)
def test_initial_biases_are_the_recorded_draws(source):
    g = film(source) if source in ('EE', 'SREE') else cases()[source]
    _, _, Bu, Bi = initial(g)
    assert np.array_equal(Bu, g['Bu0']) and np.array_equal(Bi, g['Bi0'])


def test_recorded_runs_use_the_shipped_settings():
    ee, sree = film('EE'), film('SREE')
    assert [conf_value(ee, 'reg.lambda', k) for k in ('-u', '-i', '-b')] == [0.005] * 3
    assert float(ee['lrate'][0][0]) == 0.005 and _d(ee) == 10
    assert [conf_value(sree, 'reg.lambda', k) for k in ('-u', '-i', '-b')] == [0.01] * 3
    assert float(sree['lrate'][0][0]) == 0.01 and conf_value(sree, 'SREE', '-alpha') == 0.5 and _d(sree) == 10
    assert 'item.ranking=on -topN 10' in str(sree['rank_conf'])
    assert len(sree['rank_rec_items']) > 100 and sree['rank_measure'].tolist()[0] == 'Top 10'


def test_constructed_social_file_holds_every_edge_case():
    g = cases()['sree_w']
    users, items, _, _ = load_run(g)
    visit, _, _, followees = social_of(g)
    pos = {v: k for k, v in enumerate(visit)}
    raw = list(zip(g['raw_u1'].tolist(), g['raw_u2'].tolist(), g['raw_w'].tolist()))
    assert followees['u1']['u2'] != followees['u2']['u1']                     # mutual, two weights
    assert 'u1' in followees['u1']                                            # self-follow
    assert any(w == 0 for f in followees.values() for w in f.values())        # zero-weight followee
    assert pos[users['u5']] > pos[users['u3']] and 'u5' in followees['u3']    # followee visited after its follower
    assert pos[users['u3']] < pos[users['u7']] and 'u3' in followees['u7']    # ... and one visited before
    assert raw[0][0] not in users and g['social_user'].tolist()[0] == raw[0][0]
    assert any(b not in users for _, b, _ in raw)                             # a followee who is no training user
    assert 'u8' in users and 'u8' not in g['social_user'].tolist()
    assert any(un not in users for un in g['test_users'].tolist())
    assert any(it not in items for it in g['test_items'].tolist())
    assert set(cases()['sree_nw']['raw_w'].tolist()) == {1.0}


# ------------------------------------------------------------------------------------------------ host shim
@pytest.fixture(scope='module')
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libee_sree_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'ee_sree_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    dp, i, d = C.POINTER(C.c_double), C.c_int, C.c_double
    lib.host_ee_rating_f64.argtypes = [dp, dp, i, d, d, d, dp, dp, d, d, d, d]
    lib.host_ee_rating_f64.restype = d
    lib.host_sree_user_f64.argtypes = [dp, i, dp, dp, C.POINTER(C.c_int), i, d, d]
    lib.host_sree_user_f64.restype = d
    return lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_kind5_step_source_equals_python_floats(shim):
    rs = np.random.RandomState(7)
    for _ in range(50):
        d = int(rs.randint(1, 9))
        p, q = rs.rand(d), rs.rand(d)
        r, gm, bu, bi = 0.5 * rs.randint(1, 9), 3 * rs.rand(), rs.rand() / 10, rs.rand() / 10
        lr, reg_u, reg_i, reg_b = rs.rand() / 10, rs.rand() / 10, rs.rand() / 10, rs.rand() / 10
        dist = 0.0
        for c in range(d):
            dist = dist + (float(p[c]) - float(q[c])) * (float(p[c]) - float(q[c]))
        hp, hq, hbu, hbi = p.copy(), q.copy(), np.array([bu]), np.array([bi])
        term = shim.host_ee_rating_f64(_dp(hp), _dp(hq), d, dist, r, gm, _dp(hbu), _dp(hbi), lr, reg_u, reg_i, reg_b)
        e = r - (((gm + bi) + bu) - dist)
        assert term == e * e + reg_u * dist
        for c in range(d):
            pn = float(p[c]) - (lr * (e + reg_u)) * (float(p[c]) - float(q[c]))
            assert hp[c] == pn
            assert hq[c] == float(q[c]) + (lr * (e + reg_i)) * (pn - float(q[c]))
        assert hbu[0] == bu + lr * (e - reg_b * bu) and hbi[0] == bi + lr * (e - reg_b * bi)


def test_sree_user_source_equals_python_floats(shim):
    rs = np.random.RandomState(8)
    for n in [0, 1, 2, 3, 7]:
        d = int(rs.randint(1, 9))
        p, rows = rs.randn(d), rs.randn(max(n, 1), d)
        w = np.round(rs.rand(n), 2)
        if n > 1:
            w[1] = 0.0                                                     # a zero weight
        is_self = np.array([k == n - 1 and n > 2 for k in range(max(n, 1))], np.int32)   # a self-follow last
        lr, alpha = rs.rand() / 10, rs.rand()
        hp = p.copy()
        got = shim.host_sree_user_f64(_dp(hp), d, _dp(np.ascontiguousarray(rows)), _dp(w),
                                      is_self.ctypes.data_as(C.POINTER(C.c_int)), n, lr, alpha)
        row, loss = [float(x) for x in p], 0.0
        for k in range(n):
            z = list(row) if is_self[k] else [float(x) for x in rows[k]]
            row = [row[c] - ((lr * alpha) * float(w[k])) * (row[c] - z[c]) for c in range(d)]
            sq = 0.0
            for c in range(d):
                sq = sq + (row[c] - z[c]) * (row[c] - z[c])
            loss = loss + (alpha * float(w[k])) * sq
        assert hp.tolist() == row
        assert got == loss


# ------------------------------------------------------------------------------------------------ wrappers
def wrapper_cases(torch, device):
    """(valid sree_user_pass kwargs, the invalid calls) on `device`.  Each invalid call is (call, a regex of the
    QRecError it must raise, True if the check needs the tensors' contents and so only runs on CUDA tensors)."""
    from qrec_b200 import engine as E
    U, d = 4, 5
    f64, i32, i64 = torch.float64, torch.int32, torch.int64

    def t(a, dt):
        return torch.tensor(a, dtype=dt, device=device)

    followees, followers = [[1], [0, 2], [], [3]], [[1], [0], [1], [3]]
    fr, fc = _csr(followees)
    gr, gc = _csr(followers)
    visit = np.array([3, 1, 0], np.int32)
    pos, _ = E.social_order_prepare(visit, U, fr, fc, gr, gc)
    ok = dict(P=torch.rand(U, d, dtype=f64, device=device), visit=t(visit, i32), pos=t(pos, i32), f_rowptr=t(fr, i64),
              f_cols=t(fc, i32), f_w=t([0.5, 0.25, 0.75, 1.0], f64), g_rowptr=t(gr, i64), g_cols=t(gc, i32), lr=0.05,
              alpha=0.5, loss=torch.zeros(1, dtype=f64, device=device))

    def sp(**kw):
        return lambda: E.sree_user_pass(**dict(ok, **kw))

    cases = [
        (sp(P=ok['P'].int()), 'sree_user_pass: P must be a 2-D float32 or float64 table', False),
        (sp(P=torch.zeros(U, 257, dtype=f64, device=device)), r'd=257 unsupported', False),
        (sp(visit=t([0, 1, 2, 3, 0], i32)), 'list at most 4 users', False),
        (sp(pos=t(pos[:-1], i32)), r'pos needs one entry per user \(4\)', False),
        (sp(f_rowptr=t(fr[:-1], i64)), 'the followee rowptr needs 5 entries', False),
        (sp(g_rowptr=t(gr[:-1], i64)), 'the follower rowptr needs 5 entries', False),
        (sp(f_w=t([0.5, 0.25, 0.75], f64)), 'followee ids and values differ in length', False),
        (sp(f_w=t([0.5, 0.25, 0.75, 1.0], torch.float32)), 'f_val must be torch.float64', False),
        (sp(visit=t(visit, i64)), 'visit must be torch.int32', False),
        (sp(g_rowptr=t(gr, i32)), 'g_rowptr must be torch.int64', False),
        (sp(g_cols=t(gc, i64)), 'g_cols must be torch.int32', False),
        (sp(loss=torch.zeros(0, dtype=f64, device=device)), 'loss needs one entry', False),
        (sp(loss=torch.zeros(1, dtype=torch.float32, device=device)), 'loss must be torch.float64', False),
        # contents: on CUDA tensors only, since the device check comes first
        (sp(visit=t([3, 1, 4], i32)), r'sree_user_pass: a visited user is outside \[0, 4\)', True),
        (sp(f_rowptr=t([0, 1, 3, 3, 5], i64)), 'the followee rowptr must rise from 0 to len = 4', True),
        (sp(g_rowptr=t([0, 2, 1, 3, 4], i64)), 'the follower rowptr must rise from 0 to len = 4', True),
        (sp(f_cols=t([1, 0, 2, 4], i32)), r'a followee is outside \[0, 4\)', True),
        (sp(g_cols=t([1, -1, 1, 3], i32)), r'a follower is outside \[0, 4\)', True),
        (sp(pos=t([2, 1, 0, 0], i32)), 'pos does not match the visiting order', True),
    ]
    return ok, cases


def test_sree_wrapper_checks_shapes_and_dtypes_before_touching_the_device():
    """Shapes, lengths, dtypes and d are checked before the device check, so they raise their own QRecError on CPU
    tensors; a valid call gets as far as the device check."""
    import torch
    from qrec_b200 import engine as E
    ok, bad = wrapper_cases(torch, 'cpu')
    with pytest.raises(E.QRecError, match='sree_user_pass: P must be a CUDA tensor'):
        E.sree_user_pass(**ok)
    for k, (call, message, contents) in enumerate(bad):
        if contents:
            continue
        with pytest.raises(E.QRecError, match=message):
            call()
            pytest.fail('case %d did not raise' % k)


def _kind5_args(torch, **kw):
    P = torch.zeros(2, 3, dtype=torch.float64)
    z = torch.zeros(1, dtype=torch.int32)
    args = dict(kind=5, P=P, Q=P, u=z, i=z, r=torch.zeros(1, dtype=torch.float64), wu=z, wi=z, lr=0.1, reg_u=0.1,
                reg_i=0.1, loss=torch.zeros(1, dtype=torch.float64))
    args.update(kw)
    return args


def test_mf_sgd_ordered_kind5_needs_both_bias_vectors():
    import torch
    from qrec_b200 import engine as E
    b = torch.zeros(2, dtype=torch.float64)
    assert E.EE_RATINGS == 5
    for kw in ({}, dict(Bu=b), dict(Bi=b)):
        with pytest.raises(E.QRecError, match=r'kind 5 \(EE ratings\) needs the bias vectors'):
            E.mf_sgd_ordered(**_kind5_args(torch, **kw))
    with pytest.raises(E.QRecError, match='must be a CUDA tensor'):
        E.mf_sgd_ordered(**_kind5_args(torch, Bu=b, Bi=b))


def test_dropins_keep_the_reference_surface():
    """EE and SREE resolve by name, keep the reference's constructors and rank on the host (no device_tables)."""
    import inspect
    from qrec_b200.QRec import _model_class
    from qrec_b200.base.recommender import Recommender
    ee, sree = _model_class('EE'), _model_class('SREE')
    assert list(inspect.signature(ee.__init__).parameters) == ['self', 'conf', 'trainingSet', 'testSet', 'fold']
    assert list(inspect.signature(sree.__init__).parameters) == ['self', 'conf', 'trainingSet', 'testSet', 'relation',
                                                                 'fold']
    for cls in (ee, sree):
        assert cls.device_tables is Recommender.device_tables
        assert cls.trainModel_tf is Recommender.trainModel_tf
