"""SoRec and RSTE without a GPU: the numpy oracle against the reference's golden runs, RSTE's wait numbers against a
pure-Python count, the device step source compiled on the host, and the engine wrappers' input checks."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import sorec_rste_oracle as SR     # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
RSTE_REG = dict(reg_u=0.001, reg_i=0.001, alpha=0.6)


def load_run(g):
    """ids, cleaned social structures and the training arrays of one recorded run (a dict of arrays)."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    rel = [(a, b, w) for a, b, w in zip(g['rel_u1'].tolist(), g['rel_u2'].tolist(), g['rel_w'].tolist())]
    followees, followers, kept = SR.clean_social(users, rel)
    assert kept == rel
    u0 = np.array([users[x] for x in g['train_users'].tolist()], np.int32)
    i0 = np.array([items[x] for x in g['train_items'].tolist()], np.int32)
    return users, items, rel, followees, followers, u0, i0


def conf_value(g, key, opt):
    for line in str(g['conf']).splitlines():
        if line.startswith(key + '='):
            parts = line.split('=', 1)[1].split()
            return float(parts[parts.index(opt) + 1])
    raise KeyError(key)


def replay(g, name, dtype=np.float64, epochs=None):
    """Runs the oracle over the recorded visiting orders; returns (tables after epoch 1, after the last epoch,
    losses, learning rates)."""
    users, items, rel, followees, followers, u0, i0 = load_run(g)
    tables = [t.astype(dtype) for t in SR.initial_tables(int(g['seed']), len(users), len(items), _d(g),
                                                          name == 'SoRec')]
    lr, last = float(g['lrate'][0][0]), 0.0
    losses, lrs, first = [], [], None
    eu, ev, et = SR.sorec_edges(users, followees, followers, rel)
    fl = SR.followee_lists(g['user_names'].tolist(), users, followees)
    reg_u, reg_i = conf_value(g, 'reg.lambda', '-u'), conf_value(g, 'reg.lambda', '-i')
    visits = orders(g)
    for e in range(len(visits) if epochs is None else epochs):
        o = visits[e]
        if name == 'SoRec':
            loss = SR.sorec_epoch(*tables, u0[o], i0[o], g['train_rating'][o], eu, ev, et, lr, reg_u, reg_i,
                                  conf_value(g, 'reg.lambda', '-s'), conf_value(g, 'SoRec', '-z'))
        else:
            loss = SR.rste_epoch(*tables, u0[o], i0[o], g['train_rating'][o], fl, lr, reg_u, reg_i,
                                 conf_value(g, 'RSTE', '-alpha'))
        losses.append(loss)
        before = lr
        if not abs(last - loss) < 1e-3:
            lr = SR.update_learning_rate(lr, 1.0, e + 1, last, loss)
        lrs.append((before, lr))
        last = loss
        if e == 0:
            first = [t.copy() for t in tables]
    return first, tables, losses, lrs


def orders(g):
    """Each epoch's visiting order, as indices into the initial training list: the file order first, then the list as
    isConverged's `shuffle` left it, replayed with CPython's generator from the recorded state.  The generator state
    after every shuffle must be the recorded one."""
    from oracle import bpr_oracle as O
    rng = O.make_rng(state625=g['mt_state_before'])
    order, out = list(range(len(g['train_users']))), []
    for e in range(g['lrate'].shape[0]):
        out.append(np.array(order, np.int32))
        rng.shuffle(order)
        assert np.array_equal(O.rng_state(rng), g['mt_state_after_epoch'][e])
    return out


def _d(g):
    for line in str(g['conf']).splitlines():
        if line.startswith('num.factors='):
            return int(line.split('=')[1])


def film(name):
    return dict(np.load(os.path.join(GOLD, '%s_filmtrust.npz' % name.lower())))


def cases():
    z = np.load(os.path.join(GOLD, 'social_rating_cases.npz'))
    out = {}
    for tag in z['tags'].tolist():
        out[tag] = {k.split('/', 1)[1]: z[k] for k in z.files if k.startswith(tag + '/')}
    return out


def _check_replay(g, name):
    first, tables, losses, lrs = replay(g, name)
    names = ('P', 'Q', 'Z') if name == 'SoRec' else ('P', 'Q')
    for t, k in zip(tables, names):
        assert np.array_equal(t, g[k + '_last']), k
    for t, k in zip(first, names):
        assert np.array_equal(t.astype(np.float32), g[k + '_epoch1']), k
    assert losses == g['loss'].tolist()
    assert np.array_equal(np.array(lrs), g['lrate'])


@pytest.mark.parametrize('name', ['SoRec', 'RSTE'])
def test_oracle_reproduces_the_filmtrust_run_bit_for_bit(name):
    _check_replay(film(name), name)


@pytest.mark.parametrize('tag', ['sorec_w', 'rste_w', 'rste_rank', 'sorec_nw', 'rste_nw'])
def test_oracle_reproduces_the_constructed_runs_bit_for_bit(tag):
    _check_replay(cases()[tag], 'SoRec' if tag.startswith('sorec') else 'RSTE')


@pytest.mark.parametrize('name', ['SoRec', 'RSTE'])
def test_oracle_predictions_give_the_recorded_measure(name):
    """The last tables' test predictions (RSTE: its own blend; SoRec: P.Q), clipped as checkRatingBoundary does,
    are the raw predictions the reference wrote."""
    g = film(name)
    users, items, rel, followees, _, _, _ = load_run(g)
    fl = SR.followee_lists(g['user_names'].tolist(), users, followees)
    P, Q = g['P_last'], g['Q_last']
    lo, hi = g['train_rating'].min(), g['train_rating'].max()
    checked = 0
    for k, (un, it) in enumerate(zip(g['test_users'].tolist(), g['test_items'].tolist())):
        if un not in users or it not in items:
            continue
        uu, ii = users[un], items[it]
        pred = SR.rste_predict(P, Q, uu, ii, fl, RSTE_REG['alpha']) if name == 'RSTE' else P[uu].dot(Q[ii])
        want = hi if pred > hi else lo if pred < lo else round(pred, 3)    # checkRatingBoundary
        assert g['test_pred'][k] == want, k
        checked += 1
    assert checked > 1000


def test_constructed_social_file_holds_every_edge_case():
    c = cases()['rste_w']
    users = {n: k for k, n in enumerate(c['user_names'].tolist())}
    rel = list(zip(c['rel_u1'].tolist(), c['rel_u2'].tolist(), c['rel_w'].tolist()))
    followees, _, _ = SR.clean_social(users, rel)
    assert ('u1', 'u1', 0.5) in rel                                    # self-follow
    assert [r for r in rel if r[:2] == ('u2', 'u3')] == [('u2', 'u3', 0.4), ('u2', 'u3', 0.9)]
    assert followees['u2']['u3'] == 0.9                                # the last weight wins ...
    assert list(followees['u2']) == ['u3']
    assert 'u9' not in users and all(r[1] != 'u9' for r in rel)        # cleaned away
    assert sum(followees['u4'].values()) == 0                          # denom == 0
    assert 'u8' in users and 'u8' not in followees                     # follows nobody
    tu, ti = c['test_users'].tolist(), c['test_items'].tolist()
    assert any(x not in users for x in tu) and any(x not in c['item_names'].tolist() for x in ti)
    nw = cases()['rste_nw']
    assert set(nw['rel_w'].tolist()) == {1.0}


# ------------------------------------------------------------------------------------------------ wait numbers
def _random_stream(rs, U, I, n, max_deg):
    followees = []
    for a in range(U):
        deg = rs.randint(0, max_deg + 1) if rs.rand() < 0.7 else 0
        f = list(rs.choice(U, size=min(deg, U), replace=False))
        followees.append([int(x) for x in f])
    followees[0] = [0] + [x for x in followees[0] if x != 0]          # a self-follow
    followees[1] = []                                                  # an empty list
    u = rs.randint(0, U, size=n).astype(np.int32)
    u[: n // 4] = 2                                                    # a repeated user
    i = rs.randint(0, I, size=n).astype(np.int32)
    rowptr = np.zeros(U + 1, np.int64)
    rowptr[1:] = np.cumsum([len(f) for f in followees])
    cols = np.array([x for f in followees for x in f], np.int32)
    return followees, u, i, rowptr, cols


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_rste_order_prepare_matches_pure_python(seed):
    from qrec_b200 import engine as E
    rs = np.random.RandomState(seed)
    U, I, n = 17, 9, 400
    followees, u, i, rowptr, cols = _random_stream(rs, U, I, n, 6)
    wu, wi, wr, pos_rowptr, pos, depth = E.rste_order_prepare(u, i, U, I, rowptr, cols)
    pwu, pwi, pwr, pfw, pdepth = SR.rste_waits(u, i, followees)
    assert wu.tolist() == pwu and wi.tolist() == pwi and wr.tolist() == pwr and depth == pdepth
    for a in range(U):
        assert pos[pos_rowptr[a]:pos_rowptr[a + 1]].tolist() == np.flatnonzero(u == a).tolist()
    for k in range(n):                                                 # the kernel's bisection count per followee
        others = [f for f in followees[u[k]] if f != u[k]]
        got = [int(np.searchsorted(pos[pos_rowptr[f]:pos_rowptr[f + 1]], k)) for f in others]
        assert got == pfw[k]


def test_rste_order_prepare_rejects_bad_input():
    from qrec_b200 import engine as E
    u, i = np.array([0, 1, 2], np.int32), np.array([0, 1, 0], np.int32)
    rowptr, cols = np.array([0, 1, 2, 2], np.int64), np.array([1, 0], np.int32)
    E.rste_order_prepare(u, i, 3, 2, rowptr, cols)
    bad = [(np.array([0, 3, 1], np.int32), i, rowptr, cols),           # user id out of range
           (u, np.array([0, 2, 0], np.int32), rowptr, cols),           # item id out of range
           (u, i, np.array([0, 1, 2], np.int64), cols),                # rowptr too short
           (u, i, np.array([0, 2, 1, 2], np.int64), cols),             # falling rowptr
           (u, i, np.array([1, 1, 2, 2], np.int64), cols),             # rowptr not from 0
           (u, i, rowptr, np.array([1, 3], np.int32)),                 # followee out of range
           (u, i, np.array([0, 1, 2, 3], np.int64), cols),             # rowptr past the followee list
           (np.array([0, 1], np.int32), i, rowptr, cols)]              # u and i differ in length
    for bu, bi, br, bc in bad:
        with pytest.raises(E.QRecError):
            E.rste_order_prepare(bu, bi, 3, 2, br, bc)


# ------------------------------------------------------------------------------------------------ host shim
@pytest.fixture(scope='module')
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libsocial_rating_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'social_rating_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    dp = C.POINTER(C.c_double)
    lib.host_sorec_edge_f64.restype = C.c_double
    lib.host_sorec_edge_f64.argtypes = [dp, dp, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double]
    lib.host_rste_prediction_f64.restype = C.c_double
    lib.host_rste_prediction_f64.argtypes = [C.c_double, dp, dp, C.c_int, C.c_double, C.c_double]
    return lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_kind3_step_source_equals_python_floats(shim):
    rs = np.random.RandomState(4)
    for _ in range(50):
        d = int(rs.randint(1, 9))
        p, z = rs.rand(d), rs.rand(d)
        err, lr, reg_s, reg_z = rs.randn(), rs.rand() / 10, rs.rand(), rs.rand()
        hp, hz = p.copy(), z.copy()
        term = shim.host_sorec_edge_f64(_dp(hp), _dp(hz), d, err, lr, reg_s, reg_z)
        g = reg_s * err
        for c in range(d):
            pn = float(p[c]) + lr * (g * float(z[c]))
            zn = float(z[c]) + lr * (g * pn - reg_z * float(z[c]))
            assert hp[c] == pn and hz[c] == zn
        assert term == reg_s * (err * err)


def test_rste_blend_source_equals_python_floats(shim):
    rs = np.random.RandomState(5)
    for n in [0, 1, 2, 3, 7, 20]:
        for denom_zero in (False, True):
            dot, alpha = rs.randn(), rs.rand()
            w, fd = rs.rand(n), rs.randn(n)
            denom = 0.0 if denom_zero else float(np.array(w).sum())
            got = shim.host_rste_prediction_f64(dot, _dp(w), _dp(fd), n, alpha, denom)
            s = 0.0
            for k in range(n):
                s = s + float(w[k]) * float(fd[k])
            want = dot if denom == 0 else alpha * dot + (1 - alpha) * s / denom
            assert got == want


# ------------------------------------------------------------------------------------------------ wrappers
def wrapper_cases(torch, device):
    """(valid rste_sgd_ordered kwargs, valid rste_predict_pairs kwargs, valid kind-3 mf_sgd_ordered args, the invalid
    calls) on `device`.  Each invalid call is (call, a regex of the QRecError it must raise, True if the check needs
    the tensors' contents and so only runs on CUDA tensors)."""
    from qrec_b200 import engine as E
    U, I, d, n = 4, 3, 5, 6
    f64, i32, i64 = torch.float64, torch.int32, torch.int64

    def t(a, dt):
        return torch.tensor(a, dtype=dt, device=device)

    P, Q = torch.rand(U, d, dtype=f64, device=device), torch.rand(I, d, dtype=f64, device=device)
    u, i = t([0, 1, 2, 3, 0, 1], i32), t([0, 1, 2, 0, 1, 2], i32)
    f_rowptr, f_cols, f_w = t([0, 1, 2, 2, 3], i64), t([1, 0, 2], i32), t([0.5, 1.0, 2.0], f64)
    denom = t([0.5, 1.0, 0.0, 2.0], f64)
    wu, wi, wr, pos_rowptr, pos, _ = E.rste_order_prepare(u.cpu().numpy(), i.cpu().numpy(), U, I, f_rowptr.cpu().numpy(),
                                                          f_cols.cpu().numpy())
    sgd_ok = dict(P=P, Q=Q, u=u, i=i, r=t([1.0, 2.0, 3.0, 4.0, 1.5, 2.5], f64), wu=t(wu, i32), wi=t(wi, i32),
                  wr=t(wr, i32), pos_rowptr=t(pos_rowptr, i64), pos=t(pos, i32), f_rowptr=f_rowptr, f_cols=f_cols,
                  f_w=f_w, denom=denom, lr=0.01, reg_u=0.01, reg_i=0.01, alpha=0.6,
                  loss=torch.zeros(1, dtype=f64, device=device))
    pred_ok = dict(P=P, Q=Q, u=u, i=i, f_rowptr=f_rowptr, f_cols=f_cols, f_w=f_w, denom=denom, alpha=0.6)
    Z = torch.rand(U, d, dtype=f64, device=device)
    ev = t([1, 0, 2, 3, 3, 2], i32)
    ewu, ewv = E.mf_order_prepare(u.cpu().numpy(), ev.cpu().numpy(), U, U)
    edge_ok = (3, P, Z, u, ev, sgd_ok['r'], t(ewu, i32), t(ewv, i32), 0.01, 0.1, 0.1, sgd_ok['loss'])

    def sgd(**kw):
        return lambda: E.rste_sgd_ordered(**dict(sgd_ok, **kw))

    def pred(**kw):
        return lambda: E.rste_predict_pairs(**dict(pred_ok, **kw))

    def edge(k, v, **kw):
        a = list(edge_ok)
        a[k] = v
        return lambda: E.mf_sgd_ordered(*a, **kw)

    cases = [
        (sgd(P=P.float()), 'P and Q must be float32 or float64 tables of one dtype', False),
        (sgd(P=torch.zeros(U, 257, dtype=f64, device=device), Q=torch.zeros(I, 257, dtype=f64, device=device)),
         r'd=257 unsupported', False),
        (sgd(P=torch.zeros(U, 0, dtype=f64, device=device), Q=torch.zeros(I, 0, dtype=f64, device=device)),
         r'd=0 unsupported', False),
        (sgd(Q=torch.zeros(I, d + 1, dtype=f64, device=device)), 'tables of one width', False),
        (sgd(denom=torch.zeros(U + 1, dtype=f64, device=device)), r'denom needs one entry per user \(4\), got 5', False),
        (sgd(f_rowptr=t([0, 1, 2, 2], i64)), 'the followee rowptr needs 5 entries', False),
        (sgd(f_w=t([1.0, 1.0], f64)), 'followee ids and weights differ in length', False),
        (sgd(r=torch.zeros(n + 1, dtype=f64, device=device)), 'must all hold 6 entries', False),
        (sgd(wr=t(wr[:-1], i32)), 'must all hold 6 entries', False),
        (sgd(pos=t(pos[:-1], i32)), 'must all hold 6 entries', False),
        (sgd(pos_rowptr=t(pos_rowptr[:-1], i64)), 'pos_rowptr needs 5 entries', False),
        (sgd(r=sgd_ok['r'].float()), 'r must be torch.float64, got torch.float32', False),
        (sgd(wu=sgd_ok['wu'].long()), 'wu must be torch.int32', False),
        (sgd(pos_rowptr=sgd_ok['pos_rowptr'].int()), 'pos_rowptr must be torch.int64', False),
        (sgd(f_cols=f_cols.long()), 'f_cols must be torch.int32', False),
        (pred(denom=denom[:-1]), r'denom needs one entry per user \(4\), got 3', False),
        (pred(i=t([0, 1, 2, 0, 1, 2, 0], i32)), 'u and i differ in length', False),
        (pred(Q=Q.float()), 'P and Q must be float32 or float64 tables of one dtype', False),
        (pred(out=torch.zeros(n + 1, dtype=f64, device=device)), 'out needs 6 entries', False),
        (edge(10, 0.1, Bu=torch.zeros(U, dtype=f64, device=device), Bi=torch.zeros(U, dtype=f64, device=device)),
         'kind 3 .* takes no bias vectors', False),
        (edge(2, torch.zeros(U, d + 1, dtype=f64, device=device)), 'P and Z must be 2-D tables of one width', False),
        (edge(5, sgd_ok['r'].float()), 'r must be torch.float64', False),
        (edge(4, ev[:3]), 'must all hold 6 entries', False),
        (edge(3, u + U), r'an edge source is outside \[0, 4\)', False),
        (edge(4, ev - 1), r'an edge target is outside \[0, 4\)', False),
        # contents: on CUDA tensors only, since the device check comes first
        (sgd(u=u + U), r'a user id is outside \[0, 4\)', True),
        (sgd(i=i + I), r'an item id is outside \[0, 3\)', True),
        (sgd(f_rowptr=t([0, 1, 2, 2, 4], i64)), 'the followee rowptr must rise from 0 to len', True),
        (sgd(f_rowptr=t([0, 2, 1, 2, 3], i64)), 'the followee rowptr must rise from 0 to len', True),
        (sgd(f_cols=t([1, 0, U], i32)), r'a followee is outside \[0, 4\)', True),
        (sgd(pos_rowptr=t([0, 2, 1, 5, 6], i64)), 'pos_rowptr must rise from 0 to len', True),
        (sgd(pos_rowptr=t([0, 2, 3, 4, 5], i64)), 'pos_rowptr must rise from 0 to len', True),
        (pred(u=u - 1), r'a user id is outside \[0, 4\)', True),
        (pred(i=i + I), r'an item id is outside \[0, 3\)', True),
        (pred(f_rowptr=t([1, 1, 2, 2, 3], i64)), 'the followee rowptr must rise from 0 to len', True),
        (pred(f_cols=t([1, -1, 2], i32)), r'a followee is outside \[0, 4\)', True),
    ]
    return sgd_ok, pred_ok, edge_ok, cases


def test_wrappers_check_shapes_and_dtypes_before_touching_the_device():
    """Shapes, lengths, dtypes, d, denom's length and kind 3's bias vectors are checked before the device check, so
    they raise their own QRecError on CPU tensors; a valid call gets as far as the device check."""
    import torch
    from qrec_b200 import engine as E
    sgd_ok, pred_ok, edge_ok, bad = wrapper_cases(torch, 'cpu')
    for call in (lambda: E.rste_sgd_ordered(**sgd_ok), lambda: E.rste_predict_pairs(**pred_ok),
                 lambda: E.mf_sgd_ordered(*edge_ok)):
        with pytest.raises(E.QRecError, match='must be a CUDA tensor'):
            call()
    for k, (call, message, contents) in enumerate(bad):
        if contents:
            continue
        with pytest.raises(E.QRecError, match=message):
            call()
            pytest.fail('case %d did not raise' % k)


def test_sorec_edge_weight_is_the_reference_expression():
    """weight = sqrt(|followers(v)| / (|followees(u)| + |followers(v)| + 0.0)) over the cleaned dicts."""
    g = film('SoRec')
    users, _, rel, followees, followers, _, _ = load_run(g)
    eu, ev, et = SR.sorec_edges(users, followees, followers, rel)
    a, b, t = rel[0]
    assert et[0] == math.sqrt(len(followers[b]) / (len(followees[a]) + len(followers[b]) + 0.0)) * t
    assert len(eu) == len(rel) == 1631
