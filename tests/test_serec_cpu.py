"""SERec on the CPU: the float64 oracle (oracle/serec_oracle.py) against the golden run of the unmodified reference's
SERec on FilmTrust with its trust network (tests/golden/serec_filmtrust.npz, oracle/gen_golden_serec.py), the device
prior SOURCE (qrec_b200/csrc/serec_step.cuh, through tests/host_shims/serec_step_host.cpp) against the oracle, the
drop-in's printed U x I prior against numpy's print of the materialised matrix, and the drop-in's life cycle with the
kernel replaced by the oracle.

The closed form of the prior, from the golden A and the degrees, gives the golden mu rows with the reference's bits
when deg * A is the repeated sum T.dot forms, and within 1.6e-15 relative as a single product (the largest deviation
seen; the bound is 2e-15).

The reference forms its first epoch's posteriors and Grams in float32; the oracle does everything in float64 and rounds
only the stored rows.  Over three epochs from the golden seed the largest deviation seen is 2.4e-5 of the table's
largest entry on theta, 4.6e-5 on beta and 2.6e-6 on A (all in the first epoch for beta and A); the bounds below are
about three times that."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import serec_oracle as SO      # noqa: E402
from oracle import expomf_oracle as EO     # noqa: E402
from qrec_b200.model.ranking.SERec import mu_entries, mu_text   # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'serec_filmtrust.npz')
D = 20
TOL = dict(theta=7.5e-5, beta=1.4e-4, asum=8e-6)     # of each table's largest entry


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def csrs(g):
    return EO.golden_csrs(g)


def relation(g):
    return [[a, b, w] for a, b, w in zip(g['rel_u1'].tolist(), g['rel_u2'].tolist(), g['rel_w'].tolist())]


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libserec_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'serec_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    dp, i32p = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    lib.host_serec_prior.restype = None
    lib.host_serec_prior.argtypes = [dp, C.c_int64, i32p, C.c_int64, C.c_double, C.c_double, C.c_double, C.c_double,
                                     dp]
    return lib


def host_prior(host, A, deg, n_users):
    A = np.ascontiguousarray(A, dtype=np.float64)
    deg = np.ascontiguousarray(deg, dtype=np.int32)
    out = np.empty((len(deg), len(A)))
    host.host_serec_prior(A.ctypes.data_as(C.POINTER(C.c_double)), len(A), deg.ctypes.data_as(C.POINTER(C.c_int32)),
                          len(deg), SO.A_PRIOR, SO.B_PRIOR, SO.S_SOCIAL, float(n_users),
                          out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def test_closed_form_reproduces_golden_mu_rows(g):
    """The reference's mu after every epoch, for users of degree 0, 1 and the largest degree and the printed edge
    users, from A and deg alone."""
    deg, users, items, U = g['deg'], g['mu_users'], g['mu_items'], len(g['user_names'])
    assert deg[users[0]] == 0 and deg[users[1]] == 1 and deg[users[2]] == deg.max() == 57
    assert len(items) > 250 and items[-1] == len(g['item_names']) - 1
    worst, differ = 0.0, 0
    for e in range(len(g['asum_epoch'])):
        ref = g['mu_rows_epoch'][e]
        assert ref.dtype == np.float64 and ref.shape == (len(users), len(items))
        A = g['asum_epoch'][e][items]
        assert np.array_equal(SO.prior(A, deg[users], U, form='sum'), ref)
        prod = SO.prior(A, deg[users], U, form='product')
        worst = max(worst, float((np.abs(prod - ref) / ref).max()))
        differ += int((prod != ref).sum())
    assert 0 < worst <= 2e-15
    print('closed form: repeated sum bitwise, product within %.2g relative (%d entries not bitwise)' % (worst, differ))


def test_degrees_match_golden_T(g):
    assert np.array_equal(SO.degrees(g['user_names'], relation(g)), g['deg'])
    assert (g['deg'] == 0).sum() == 977 and len(set(g['deg'].tolist())) == 24


def _conf(extra=''):
    from qrec_b200.util.config import ModelConf
    return ModelConf.from_string("""ratings=r.txt
social=t.txt
ratings.setup=-columns 0 1 2
social.setup=-columns 0 1
model.name=SERec
evaluation.setup=-testSet s.txt
item.ranking=on -topN 10
num.factors=4
num.max.epoch=1
learnRate=-init 0.01 -max 1
reg.lambda=-u 1 -i 0.02 -b 0.02 -s 0.01
output.setup=off
""" + extra)


def test_degrees_follow_the_cleaned_social_view(tmp_path, monkeypatch):
    """Relations to unknown users, a user whose followees are all unknown, an unknown follower, self-follows and a
    repeated pair: the drop-in's degrees, the oracle's and the row sums of the reference's T (built statement for
    statement from the cleaned followees) agree."""
    from qrec_b200.model.ranking.SERec import SERec
    monkeypatch.chdir(tmp_path)
    train = [['u%d' % u, 'i%d' % (u % 3), 1.0] for u in range(6)]
    test = [['u0', 'i1', 1.0]]
    rel = [['u0', 'u1', 1.0], ['u0', 'u2', 0.5], ['u0', 'x9', 1.0],       # one unknown followee
           ['u1', 'x8', 1.0], ['u1', 'x7', 1.0],                           # every followee unknown
           ['x6', 'u3', 1.0],                                              # unknown follower
           ['u2', 'u2', 1.0], ['u3', 'u3', 0.2], ['u3', 'u4', 1.0],        # self-follows
           ['u4', 'u5', 1.0], ['u4', 'u5', 3.0]]                           # a repeated pair
    model = SERec(_conf(), train, test, rel)
    model.readConfiguration()
    model.initModel()
    row, col = [], []
    for user in model.social.followees:                                    # SERec.py: initModel's T
        for f in model.social.followees[user]:
            row.append(model.data.user[user])
            col.append(model.data.user[f])
    T = sp.csr_matrix((np.ones(len(row)), (row, col)), (model.num_users, model.num_users))
    names = [model.data.id2user[k] for k in range(model.num_users)]
    want = np.asarray(T.sum(axis=1)).ravel().astype(np.int32)
    assert np.array_equal(model.deg, want) and np.array_equal(SO.degrees(names, rel), want)
    assert want.tolist() == [[2, 0, 1, 2, 1, 0][int(n[1:])] for n in names]


def test_oracle_tracks_golden_epochs(g, csrs):
    theta, beta = SO.initial_state(g, D)
    A, worst = None, {}
    for e in range(len(g['asum_epoch'])):
        A, failed = SO.epoch(theta, beta, A, g['deg'], *csrs)
        assert failed == 0
        for name, got in (('theta', theta), ('beta', beta), ('asum', A)):
            ref = g[name + '_epoch'][e].astype(np.float64)
            err = float(np.abs(got.astype(np.float64) - ref).max() / np.abs(ref).max())
            worst[name] = max(worst.get(name, 0.0), err)
            assert err <= TOL[name], (name, e, err)
    print('oracle vs golden, largest deviation of scale:', worst)


def test_device_prior_source_equals_oracle(g, host):
    rng = np.random.default_rng(1)
    U = len(g['user_names'])
    deg = np.concatenate([np.arange(60), [0, 1, 57, 1000, 100000]]).astype(np.int32)
    for A in (g['asum_epoch'][0], g['asum_epoch'][-1], rng.uniform(0, U, 500), np.array([0.0, 1.0, U, 1e-300])):
        got = host_prior(host, A, deg, U)
        assert np.array_equal(got, SO.prior(A, deg, U, form='product'))


def _reference_mu(A, followees, n_users):
    """SERec.py: _update_expo's prior, literally: tile, T.dot, and the expression."""
    row = [u for u, fs in enumerate(followees) for _ in fs]
    col = [f for fs in followees for f in fs]
    T = sp.csr_matrix((np.ones(len(row), dtype=np.int64), (row, col)), (n_users, n_users))
    A_sum = np.tile(A, [n_users, 1])
    S_sum = T.dot(A_sum)
    return (1.0 + A_sum + (2.2 - 1) * S_sum - 1) / (1.0 + 99.0 + (2.2 - 1) * S_sum + n_users - 2)


@pytest.mark.parametrize('U,I', [(3, 4), (10, 100), (10, 101), (2, 2000), (2000, 2), (7, 7), (40, 40), (300, 500)])
def test_printed_mu_equals_print_of_materialised_matrix(U, I):
    """Small (not summarised), just over the threshold, one short axis, square shapes: the drop-in's text is
    str() of the reference's matrix, for the first epoch's float32 mu and for a formed one."""
    rng = np.random.default_rng(U * 7919 + I)
    followees = [sorted(set(rng.choice(U, int(rng.choice([0, 0, 1, 3, 9, 25])), replace=True).tolist()))
                 for _ in range(U)]
    deg = np.array([len(f) for f in followees], dtype=np.int32)
    A = rng.uniform(0, U, I) * rng.choice([1e-3, 1.0], I)
    assert mu_text(None, deg, I) == str(0.01 * np.ones((U, I), dtype=np.float32))
    ref = _reference_mu(A, followees, U)
    assert mu_text(A, deg, I) == str(ref)
    assert np.array_equal(mu_entries(A, deg, U), ref)


def test_printed_mu_equals_golden_prints(g):
    deg, I = g['deg'], len(g['item_names'])
    texts = g['mu_str'].tolist()
    assert texts[0] == mu_text(None, deg, I)
    for e in range(1, len(texts)):
        assert texts[e] == mu_text(g['asum_epoch'][e - 1], deg, I)


def test_square_tables_take_the_user_branch_in_the_item_half():
    """U == I: the reference's item half reads mu[i, :]; the oracle's default does the same."""
    rng = np.random.default_rng(6)
    n, d = 40, 6
    Y = (rng.random((n, n)) < 0.15)
    theta = (rng.standard_normal((n, d)) * 0.5).astype(np.float32)
    beta = (rng.standard_normal((n, d)) * 0.5).astype(np.float32)
    deg = rng.integers(0, 30, n).astype(np.int32)
    A = rng.uniform(0.5, 10, n)
    urp = np.concatenate([[0], np.cumsum(Y.sum(1))]).astype(np.int64)
    ucol = np.concatenate([np.flatnonzero(r) for r in Y]).astype(np.int32)
    irp = np.concatenate([[0], np.cumsum(Y.T.sum(1))]).astype(np.int64)
    icol = np.concatenate([np.flatnonzero(r) for r in Y.T]).astype(np.int32)
    out = {}
    for quirk in (None, True, False):
        t, b = theta.copy(), beta.copy()
        out[quirk] = (SO.epoch(t, b, A, deg, (urp, ucol), (irp, icol), square_quirk=quirk)[0], b)
    assert np.array_equal(out[None][0], out[True][0]) and np.array_equal(out[None][1], out[True][1])
    assert np.abs(out[False][1] - out[True][1]).max() > 1e-3 * np.abs(out[True][1]).max()


def test_model_class_resolves():
    from qrec_b200.QRec import _model_class
    from qrec_b200.model.ranking.SERec import SERec
    assert _model_class('SERec') is SERec


def oracle_half_epoch(X, Z, rowptr, cols, asum, deg, row_is_user, lam, lam_y, row_order, asum_out=None, mu0=0.01,
                      a=1.0, b=99.0, s=2.2, n_failed=None, max_ctas=0):
    """engine.serec_half_epoch on CPU tensors through the oracle."""
    rows = row_order.numpy()
    Xn, Zn, dn = X.numpy(), Z.numpy(), deg.numpy()
    n, m = Xn.shape[0], Zn.shape[0]
    U = n if row_is_user else m
    assert mu0 == SO.INIT_MU and (a, b, s) == (SO.A_PRIOR, SO.B_PRIOR, SO.S_SOCIAL)
    A = None if asum is None else asum.numpy()
    if A is None:
        M = Mo = np.full((n, m), SO.MU0)
    else:
        M = SO.prior(A, dn, U) if row_is_user else SO.prior(A, dn, U).T
        Mo = SO.prior(A, dn, U).T if asum_out is not None else None
    assert SO.solve_side(Xn, Zn, rowptr.numpy(), cols.numpy(), M, lam, lam_y, rows) == 0
    if asum_out is not None:
        asum_out.numpy()[rows] = SO.asum_rows(Xn, Zn, rowptr.numpy(), cols.numpy(), Mo, lam_y, rows)
    return X


def test_dropin_life_cycle_with_oracle_kernel(g, tmp_path, monkeypatch):
    """The drop-in from the golden seed with serec_half_epoch replaced by the oracle on CPU tensors: the initModel
    draws, the degrees, the printed lines, the tables after the last epoch and the ranking."""
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.iterativeRecommender import IterativeRecommender
    from qrec_b200.model.ranking.SERec import SERec
    from qrec_b200.util.config import ModelConf

    calls = []

    def half(*args, **kw):
        calls.append((args[4] is None, args[6], kw.get('asum_out') is not None))
        return oracle_half_epoch(*args, **kw)

    monkeypatch.setattr(E, 'serec_half_epoch', half)
    monkeypatch.setattr(IterativeRecommender, '_device', lambda self: torch.device('cpu'))
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']))
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    model = SERec(conf, train, test, relation(g))
    lines = []
    orig_print = print

    def spy_print(*args, **kw):
        if args and isinstance(args[0], str):
            lines.append(args[0])
        orig_print(*args, **kw)
    monkeypatch.setattr('builtins.print', spy_print)
    measure = model.execute()
    monkeypatch.undo()
    n_epochs = len(g['asum_epoch'])
    assert np.array_equal(model.deg, g['deg'])
    assert calls == [(True, True, False), (True, False, True)] + [(False, True, False), (False, False, True)] * (n_epochs - 1)
    k = lines.index('epoch #0')
    texts = g['mu_str'].tolist()
    assert lines[k:k + 3] == ['epoch #0', texts[0], '\tUpdating exposure prior...']
    for e in range(1, n_epochs):
        j = lines.index('epoch #%d' % e)
        assert lines[j + 2] == '\tUpdating exposure prior...'
        assert len(lines[j + 1].splitlines()) == len(texts[e].splitlines())     # a summarised U x I print
    assert model.theta.dtype == model.beta.dtype == np.float32
    for name, got in (('theta', model.theta), ('beta', model.beta), ('asum', model.A)):
        ref = g[name + '_epoch'][-1]
        np.testing.assert_allclose(got.astype(np.float64), ref, rtol=0, atol=TOL[name] * float(np.abs(ref).max()))
    rows = model.mu_rows(g['mu_users'])[:, g['mu_items']]
    np.testing.assert_allclose(rows, g['mu_rows_epoch'][-1], rtol=3 * TOL['asum'])
    u = g['test_users'][0]
    assert np.array_equal(model.predictForRanking(u), model.beta.dot(model.theta[model.data.getUserId(u)]))
    assert_measure(measure, g)


def assert_measure(measure, g):
    """Precision, recall, F1 and NDCG to 1e-4 of their printed values (the float64 tables may swap a pair of
    neighbours inside a top-10 list against the reference's float32 ones)."""
    assert len(measure) == len(g['measure'])
    for got, ref in zip(measure, g['measure'].tolist()):
        if ':' in ref:
            name, val = ref.split(':')
            assert got.strip().startswith(name + ':') and abs(float(got.split(':')[1]) - float(val)) < 1e-4, (got, ref)
        else:
            assert got.strip() == ref
