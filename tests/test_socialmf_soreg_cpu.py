"""SocialMF and SoReg without a GPU: the numpy oracle against the reference's golden runs and similarities, the user
pass's schedule against a pure-Python count, the device step source compiled on the host, and the engine wrappers'
input checks."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import socialmf_soreg_oracle as SM      # noqa: E402
from oracle import sorec_rste_oracle as SR          # noqa: E402
from test_social_rating_cpu import _d, conf_value, orders   # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
TAGS = ['socialmf_w', 'soreg_w', 'socialmf_nw', 'soreg_nw']


def film(name):
    return dict(np.load(os.path.join(GOLD, '%s_filmtrust.npz' % name.lower())))


def cases():
    z = np.load(os.path.join(GOLD, 'socialmf_soreg_cases.npz'))
    out = {}
    for tag in z['tags'].tolist():
        out[tag] = {k.split('/', 1)[1]: z[k] for k in z.files if k.startswith(tag + '/')}
    return out


def case_files():
    z = np.load(os.path.join(GOLD, 'socialmf_soreg_cases.npz'))
    return {k.split('/', 1)[1]: z[k] for k in z.files if k.startswith('files/')}


def load_run(g):
    """ids, the cleaned social dicts built from the relation list as read, the training rows and arrays of a run."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    raw = list(zip(g['raw_u1'].tolist(), g['raw_u2'].tolist(), g['raw_w'].tolist()))
    followees, followers, kept = SR.clean_social(users, raw)
    assert kept == list(zip(g['rel_u1'].tolist(), g['rel_u2'].tolist(), g['rel_w'].tolist()))
    first = []
    for a, b, _ in raw:
        for x in (a, b):
            if x not in first:
                first.append(x)
    assert first == g['social_user'].tolist()
    rows = {}
    for un, it, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist()):
        rows.setdefault(un, {})[it] = r
    u0 = np.array([users[x] for x in g['train_users'].tolist()], np.int32)
    i0 = np.array([items[x] for x in g['train_items'].tolist()], np.int32)
    return users, items, followees, followers, rows, u0, i0


def social_lists(g, name, sim=None):
    """(visit, followee lists, follower lists) of a run; the values are the weights (SocialMF) or Sim (SoReg)."""
    users, _, followees, followers, rows, _, _ = load_run(g)
    names = g['user_names'].tolist()
    if name == 'SoReg' and sim is None:
        sim, _ = SM.soreg_similarities(names, followees, rows)
    visit = SM.visit_ids(g['social_user'].tolist(), users)
    return visit, SM.neighbour_lists(names, users, followees, sim), SM.neighbour_lists(names, users, followers, sim)


def replay(g, name, dtype=np.float64):
    """The oracle over the recorded visiting orders: (tables after epoch 1, after the last epoch, losses, rates)."""
    users, items, _, _, _, u0, i0 = load_run(g)
    P, Q = (t.astype(dtype) for t in SR.initial_tables(int(g['seed']), len(users), len(items), _d(g), False))
    visit, fl, gl = social_lists(g, name)
    reg_u, reg_i = conf_value(g, 'reg.lambda', '-u'), conf_value(g, 'reg.lambda', '-i')
    lr, last = float(g['lrate'][0][0]), 0.0
    losses, lrs, first = [], [], None
    for e, o in enumerate(orders(g)):
        args = (P, Q, u0[o], i0[o], g['train_rating'][o], visit, fl)
        if name == 'SocialMF':
            loss = SM.socialmf_epoch(*args, lr, reg_u, reg_i, conf_value(g, 'reg.lambda', '-s'))
        else:
            loss = SM.soreg_epoch(*args, gl, lr, reg_u, reg_i, conf_value(g, 'SoReg', '-alpha'))
        losses.append(loss)
        before = lr
        if not abs(last - loss) < 1e-3:
            lr = SR.update_learning_rate(lr, 1.0, e + 1, last, loss)
        lrs.append((before, lr))
        last = loss
        if e == 0:
            first = (P.copy(), Q.copy())
    return first, (P, Q), losses, lrs


def predictions(g, P, Q):
    """Each test line's prediction from the tables, with iterativeRecommender's fallbacks, clipped as
    checkRatingBoundary does; and the measure lines of that list."""
    from qrec_b200.util.measure import Measure
    users, items, _, _, rows, _, _ = load_run(g)
    user_means = {u: sum(r.values()) / len(r) for u, r in rows.items()}
    cols = {}
    for un, it, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist()):
        cols.setdefault(it, {})[un] = r
    item_means = {i: sum(c.values()) / len(c) for i, c in cols.items()}
    total = sum(user_means.values())
    global_mean = total / len(user_means) if total != 0 else 0
    lo, hi = min(g['train_rating']), max(g['train_rating'])
    res = []
    for un, it, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist()):
        if un in users and it in items:
            pred = P[users[un]].dot(Q[items[it]])
        else:
            pred = user_means[un] if un in users else item_means[it] if it in items else global_mean
        res.append([un, it, r, hi if pred > hi else lo if pred < lo else round(pred, 3)])
    return [x[3] for x in res], [m.strip() for m in Measure.ratingMeasure(res)]


def _check(g, name):
    first, tables, losses, lrs = replay(g, name)
    for t, k in zip(tables, 'PQ'):
        assert np.array_equal(t, g[k + '_last']), k
    for t, k in zip(first, 'PQ'):
        assert np.array_equal(t.astype(np.float32), g[k + '_epoch1']), k
    assert losses == g['loss'].tolist()
    assert np.array_equal(np.array(lrs), g['lrate'])
    preds, measure = predictions(g, *tables)
    assert preds == g['test_pred'].tolist()
    assert measure == g['measure'].tolist()


@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
def test_oracle_reproduces_the_filmtrust_run_bit_for_bit(name):
    _check(film(name), name)


@pytest.mark.parametrize('tag', TAGS)
def test_oracle_reproduces_the_constructed_runs_bit_for_bit(tag):
    _check(cases()[tag], 'SoReg' if tag.startswith('soreg') else 'SocialMF')


def _recorded_sim(g):
    return list(zip(g['sim_user'].tolist(), g['sim_friend'].tolist(), g['sim_value'].tolist()))


@pytest.mark.parametrize('source', ['film', 'soreg_w', 'soreg_nw'])
def test_oracle_similarities_equal_the_recorded_ones(source):
    g = film('SoReg') if source == 'film' else cases()[source]
    users, _, followees, _, rows, _, _ = load_run(g)
    sim, pairs = SM.soreg_similarities(g['user_names'].tolist(), followees, rows)
    got = [(a, b, v) for a in sim for b, v in sim[a].items()]
    rec = _recorded_sim(g)
    assert [x[:2] for x in got] == [x[:2] for x in rec]
    assert all(np.float64(x[2]).tobytes() == np.float64(y[2]).tobytes() for x, y in zip(got, rec))
    assert len(pairs) * 2 - sum(a == b for a, b in pairs) == len(rec)


def test_constructed_social_file_holds_every_edge_case():
    g = cases()['soreg_w']
    users, _, followees, followers, rows, _, _ = load_run(g)
    sim = dict(((a, b), v) for a, b, v in _recorded_sim(g))
    raw = list(zip(g['raw_u1'].tolist(), g['raw_u2'].tolist(), g['raw_w'].tolist()))
    assert followees['u1']['u2'] != followees['u2']['u1']                     # mutual, two weights
    assert sim[('u1', 'u2')] == sim[('u2', 'u1')]                             # ... one similarity, met first
    first = 'u1' if users['u1'] < users['u2'] else 'u2'
    other = 'u2' if first == 'u1' else 'u1'
    assert sim[('u1', 'u2')] == (SM.KO.similarity(rows[first], rows[other], 'pcc') + followees[first][other]) / 2.0
    assert len(set(rows['u5'].values())) == 1 and 'u5' in followees['u3']    # zero variance, pcc 1
    assert SM.KO.similarity(rows['u3'], rows['u5'], 'pcc') == 1
    assert not set(rows['u6']) & set(rows['u1']) and 'u1' in followees['u6']  # no co-rated item, pcc 0
    assert sum(followees['u4'].values()) == 0 and len(followees['u4']) == 2  # denom == 0
    assert 'u1' in followees['u1']                                            # self-follow
    assert raw[0][0] not in users and g['social_user'].tolist()[0] == raw[0][0]
    assert 'u8' in users and 'u8' not in g['social_user'].tolist()
    assert set(cases()['soreg_nw']['raw_w'].tolist()) == {1.0}


# ------------------------------------------------------------------------------------------------ schedule
def _random_graph(rs, U, max_deg):
    followees = [sorted(set(rs.choice(U, size=rs.randint(0, max_deg + 1)).tolist())) for _ in range(U)]
    followees[0] = [0] + [x for x in followees[0] if x != 0]           # a self-follow
    followees[1] = []
    followers = [[] for _ in range(U)]
    for a in range(U):
        for b in followees[a]:
            followers[b].append(a)
    return followees, followers


def _csr(lists):
    rowptr = np.zeros(len(lists) + 1, np.int64)
    rowptr[1:] = np.cumsum([len(x) for x in lists])
    return rowptr, np.array([v for x in lists for v in x], np.int32)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_social_order_prepare_matches_pure_python(seed):
    from qrec_b200 import engine as E
    rs = np.random.RandomState(seed)
    U = 40
    followees, followers = _random_graph(rs, U, 6)
    visit = rs.permutation(U)[:30].astype(np.int32)                   # ten users are not visited
    pos, depth = E.social_order_prepare(visit, U, *_csr(followees), *_csr(followers))
    ppos, pdepth = SM.schedule(visit.tolist(), U, followees, followers)
    assert pos.tolist() == ppos and depth == pdepth


def test_social_order_prepare_rejects_bad_input():
    from qrec_b200 import engine as E
    f = _csr([[1], [0], []])
    g = _csr([[1], [0], []])
    visit = np.array([2, 0, 1], np.int32)
    E.social_order_prepare(visit, 3, *f, *g)
    bad = [(np.array([0, 3], np.int32), f, g),                         # visit out of range
           (np.array([0, 0], np.int32), f, g),                         # a user visited twice
           (np.array([0, 1, 2, 0], np.int32), f, g),                   # longer than the user count
           (visit, (np.array([0, 1, 2], np.int64), f[1]), g),          # rowptr too short
           (visit, (np.array([0, 2, 1, 2], np.int64), f[1]), g),       # falling rowptr
           (visit, (np.array([1, 1, 2, 2], np.int64), f[1]), g),       # rowptr not from 0
           (visit, (np.array([0, 1, 2, 3], np.int64), f[1]), g),       # rowptr past the columns
           (visit, (np.array([0, 1, 1, 1], np.int64), f[1]), g),       # rowptr short of the columns
           (visit, f, (g[0], np.array([1, 3], np.int32)))]             # follower out of range
    for v, ff, gg in bad:
        with pytest.raises(E.QRecError):
            E.social_order_prepare(v, 3, *ff, *gg)


# ------------------------------------------------------------------------------------------------ host shim
@pytest.fixture(scope='module')
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libsocial_pass_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'social_pass_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    dp, i, d = C.POINTER(C.c_double), C.c_int, C.c_double
    lib.host_socialmf_rating_f64.argtypes = [dp, dp, i, d, d, d, d]
    lib.host_socialmf_user_f64.argtypes = [dp, i, dp, dp, i, d, d]
    lib.host_soreg_user_f64.argtypes = [dp, i, dp, dp, i, dp, dp, i, d, d]
    return lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_kind4_step_source_equals_python_floats(shim):
    rs = np.random.RandomState(4)
    for _ in range(50):
        d = int(rs.randint(1, 9))
        p, q = rs.rand(d), rs.rand(d)
        err, lr, reg_u, reg_i = rs.randn(), rs.rand() / 10, rs.rand(), rs.rand()
        hp, hq = p.copy(), q.copy()
        shim.host_socialmf_rating_f64(_dp(hp), _dp(hq), d, err, lr, reg_u, reg_i)
        for c in range(d):
            assert hp[c] == float(p[c]) + lr * (err * float(q[c]) - reg_u * float(p[c]))
            assert hq[c] == float(q[c]) + lr * (err * float(p[c]) - reg_i * float(q[c]))


def test_socialmf_user_source_equals_python_floats(shim):
    rs = np.random.RandomState(5)
    for n in [0, 1, 2, 3, 7]:
        for zero in (False, True):
            d = int(rs.randint(1, 9))
            p, rows = rs.randn(d), rs.randn(max(n, 1), d)
            w = np.zeros(n) if zero else rs.rand(n)
            lr, reg_s = rs.rand() / 10, rs.rand()
            hp = p.copy()
            shim.host_socialmf_user_f64(_dp(hp), d, _dp(np.ascontiguousarray(rows)), _dp(w), n, lr, reg_s)
            denom = 0.0
            for k in range(n):
                denom = denom + float(w[k])
            for c in range(d):
                want = float(p[c])
                if denom != 0:
                    f = 0.0
                    for k in range(n):
                        f = f + float(w[k]) * float(rows[k, c])
                    want = float(p[c]) - (lr * reg_s) * (float(p[c]) - f / denom)
                assert hp[c] == want


def test_soreg_user_source_equals_python_floats(shim):
    rs = np.random.RandomState(6)
    for nf, ng in [(0, 0), (1, 0), (0, 2), (3, 4), (7, 1)]:
        d = int(rs.randint(1, 9))
        p, fr, gr = rs.randn(d), rs.randn(max(nf, 1), d), rs.randn(max(ng, 1), d)
        fs, gs = rs.randn(nf), rs.randn(ng)
        lr, alpha = rs.rand() / 10, rs.rand()
        hp = p.copy()
        shim.host_soreg_user_f64(_dp(hp), d, _dp(np.ascontiguousarray(fr)), _dp(fs), nf, _dp(np.ascontiguousarray(gr)),
                                 _dp(gs), ng, lr, alpha)
        for c in range(d):
            f1 = f2 = 0.0
            for k in range(nf):
                f1 = f1 + float(fs[k]) * (float(p[c]) - float(fr[k, c]))
            for k in range(ng):
                f2 = f2 + float(gs[k]) * (float(p[c]) - float(gr[k, c]))
            assert hp[c] == float(p[c]) + lr * (-alpha * (f1 + f2))


# ------------------------------------------------------------------------------------------------ wrappers
def wrapper_cases(torch, device):
    """(valid social_user_pass kwargs for kind 1, valid knn_pair_similarity args, the invalid calls) on `device`.  Each
    invalid call is (call, a regex of the QRecError it must raise, True if the check needs the tensors' contents and so
    only runs on CUDA tensors)."""
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
    pass_ok = dict(kind=1, P=torch.rand(U, d, dtype=f64, device=device), visit=t(visit, i32), pos=t(pos, i32),
                   f_rowptr=t(fr, i64), f_cols=t(fc, i32), f_val=t([0.5, 0.25, 0.75, 1.0], f64), g_rowptr=t(gr, i64),
                   g_cols=t(gc, i32), g_val=t([0.5, 0.25, 0.75, 1.0], f64), lr=0.05, coef=0.1,
                   loss=torch.zeros(1, dtype=f64, device=device))
    rowptr, cols = t([0, 2, 3, 5], i64), t([1, 0, 2, 0, 1], i32)
    vals = t([3.0, 4.0, 2.0, 1.0, 5.0], f64)
    sim_ok = dict(rowptr=rowptr, cols=cols, vals=vals, sq=vals * 0.5, means=t([3.5, 2.0, 3.0], f64),
                  sorted_cols=t([0, 1, 2, 0, 1], i32), sorted_vals=t([4.0, 3.0, 2.0, 1.0, 5.0], f64),
                  sorted_sq=t([2.0, 1.5, 1.0, 0.5, 2.5], f64), a=t([0, 2], i32), b=t([2, 1], i32), w=t([0.5, 1.0], f64))

    def sp(**kw):
        return lambda: E.social_user_pass(**dict(pass_ok, **kw))

    def ps(**kw):
        return lambda: E.knn_pair_similarity(**dict(sim_ok, **kw))

    cases = [
        (sp(kind=2), 'kind must be 0 .SocialMF. or 1 .SoReg.', False),
        (sp(g_val=None), 'SoReg needs the followers', False),
        (sp(P=pass_ok['P'].int()), 'P must be a 2-D float32 or float64 table', False),
        (sp(P=torch.zeros(U, 257, dtype=f64, device=device)), r'd=257 unsupported', False),
        (sp(visit=t([0, 1, 2, 3, 0], i32)), 'list at most 4 users', False),
        (sp(pos=t(pos[:-1], i32)), r'pos needs one entry per user \(4\)', False),
        (sp(f_rowptr=t(fr[:-1], i64)), 'the followee rowptr needs 5 entries', False),
        (sp(g_rowptr=t(gr[:-1], i64)), 'the follower rowptr needs 5 entries', False),
        (sp(f_val=t([0.5, 0.25, 0.75], f64)), 'followee ids and values differ in length', False),
        (sp(g_val=t([0.5], f64)), 'follower ids and values differ in length', False),
        (sp(f_val=t([0.5, 0.25, 0.75, 1.0], torch.float32)), 'f_val must be torch.float64', False),
        (sp(visit=t(visit, i64)), 'visit must be torch.int32', False),
        (sp(g_rowptr=t(gr, i32)), 'g_rowptr must be torch.int64', False),
        (sp(loss=torch.zeros(1, dtype=torch.float32, device=device)), 'loss must be torch.float64', False),
        (ps(a=t([0, 2], i64)), 'a and b must be int32 of one length', False),
        (ps(b=t([2], i32)), 'a and b must be int32 of one length', False),
        (ps(w=t([0.5], f64)), r'w must be float64 \[2\]', False),
        (ps(sq=vals[:4]), r'sq must be float64 \[5\]', False),
        (ps(means=t([3.5, 2.0], f64)), r'means must be float64 \[3\]', False),
        (ps(sorted_cols=t([0, 1, 2, 0, 1], i64)), 'cols and sorted_cols must be 1-D int32', False),
        # contents: on CUDA tensors only, since the device check comes first
        (sp(visit=t([3, 1, 4], i32)), r'a visited user is outside \[0, 4\)', True),
        (sp(f_rowptr=t([0, 1, 3, 3, 5], i64)), 'the followee rowptr must rise from 0 to len = 4', True),
        (sp(g_rowptr=t([0, 2, 1, 3, 4], i64)), 'the follower rowptr must rise from 0 to len = 4', True),
        (sp(f_cols=t([1, 0, 2, 4], i32)), r'a followee is outside \[0, 4\)', True),
        (sp(g_cols=t([1, -1, 1, 3], i32)), r'a follower is outside \[0, 4\)', True),
        (sp(pos=t([2, 1, 0, 0], i32)), 'pos does not match the visiting order', True),
        (sp(pos=t([2, 1, -1, -1], i32)), 'pos does not match the visiting order', True),
        (ps(rowptr=t([0, 2, 3, 4], i64)), 'rowptr must rise from 0 to len.cols. = 5', True),
        (ps(sorted_cols=t([1, 0, 2, 0, 1], i32)), 'sorted_cols must rise strictly within each row', True),
        (ps(a=t([0, 3], i32)), r'a row id is outside \[0, 3\)', True),
        (ps(b=t([-1, 1], i32)), r'a row id is outside \[0, 3\)', True),
    ]
    return pass_ok, sim_ok, cases


def test_wrappers_check_shapes_and_dtypes_before_touching_the_device():
    """Shapes, lengths, dtypes and d are checked before the device check, so they raise their own QRecError on CPU
    tensors; a valid call gets as far as the device check."""
    import torch
    from qrec_b200 import engine as E
    pass_ok, sim_ok, bad = wrapper_cases(torch, 'cpu')
    for call in (lambda: E.social_user_pass(**pass_ok), lambda: E.knn_pair_similarity(**sim_ok)):
        with pytest.raises(E.QRecError, match='must be a CUDA tensor'):
            call()
    for k, (call, message, contents) in enumerate(bad):
        if contents:
            continue
        with pytest.raises(E.QRecError, match=message):
            call()
            pytest.fail('case %d did not raise' % k)


def test_mf_sgd_ordered_kind4_rejects_bias_vectors():
    import torch
    from qrec_b200 import engine as E
    P = torch.zeros(2, 3, dtype=torch.float64)
    z = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(E.QRecError, match='kind 4 .SocialMF ratings. takes no bias vectors'):
        E.mf_sgd_ordered(E.SOCIALMF_RATINGS, P, P, z, z, torch.zeros(1, dtype=torch.float64), z, z, 0.1, 0.1, 0.1,
                         torch.zeros(1, dtype=torch.float64), Bu=torch.zeros(2, dtype=torch.float64),
                         Bi=torch.zeros(2, dtype=torch.float64))
