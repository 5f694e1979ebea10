"""SVD++ (K11) on the CPU: the numpy oracle (oracle/svdpp_oracle.py) against the golden run of the unmodified
reference's SVD++ on FilmTrust (tests/golden/svdpp_filmtrust.npz, oracle/gen_golden_svdpp.py), the per-user closed
form against the literal loop, the device arithmetic SOURCE (qrec_b200/csrc/svdpp_step.cuh, through
tests/host_shims/svdpp_step_host.cpp) against both, and the drop-in's life cycle with the kernel replaced by the
oracle."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import bpr_oracle as O            # noqa: E402
from oracle import svdpp_oracle as S          # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'svdpp_filmtrust.npz')
REG = dict(reg_u=0.01, reg_i=0.01, reg_b=0.1, reg_y=0.01)        # SVD++.conf
TABLES = ('P', 'Q', 'Y', 'Bu', 'Bi')


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def ids(g):
    return S.golden_ids(g)


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libsvdpp_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'svdpp_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    for name, ft, sc in (('host_svdpp_ordered_f64', C.POINTER(C.c_double), C.c_double),
                         ('host_svdpp_ordered_f32', C.POINTER(C.c_float), C.c_float)):
        fn = getattr(lib, name)
        fn.restype = C.c_double
        fn.argtypes = [ft] * 5 + [C.c_int, C.c_int64, i32, i32, ft, i64, i32] + [sc] * 6
    fn = lib.host_svdpp_usermajor_f32
    fn.restype = C.c_double
    fn.argtypes = [C.POINTER(C.c_float)] * 5 + [C.c_int, C.c_int, i32, i64, i32, C.POINTER(C.c_float)] + [C.c_float] * 6
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def host_ordered(host, tabs, u, i, r, csr, lr, gm):
    P = tabs[0]
    f64 = P.dtype == np.float64
    ft = C.c_double if f64 else C.c_float
    fn = host.host_svdpp_ordered_f64 if f64 else host.host_svdpp_ordered_f32
    rowptr, cols = csr[0], csr[1]
    r = np.ascontiguousarray(r, dtype=P.dtype)
    u, i = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(i, np.int32)
    return fn(*[_p(t, ft) for t in tabs], P.shape[1], len(u), _p(u, C.c_int32), _p(i, C.c_int32), _p(r, ft),
              _p(rowptr, C.c_int64), _p(cols, C.c_int32), lr, REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'], gm)


def host_usermajor(host, tabs, csr, order, lr, gm):
    rowptr, cols, vals = csr
    vals = np.ascontiguousarray(vals, dtype=np.float32)
    order = np.ascontiguousarray(order, np.int32)
    return host.host_svdpp_usermajor_f32(*[_p(t, C.c_float) for t in tabs], tabs[0].shape[1], len(order),
                                         _p(order, C.c_int32), _p(rowptr, C.c_int64), _p(cols, C.c_int32),
                                         _p(vals, C.c_float), lr, REG['reg_u'], REG['reg_i'], REG['reg_b'],
                                         REG['reg_y'], gm)


def rating_lines(g, tabs, csr, users, items):
    """MAE / RMSE of rating_performance (base/iterativeRecommender.py:104-113) from the tables."""
    from qrec_b200.util.measure import Measure
    P, Q, Y, Bu, Bi = tabs
    rowptr, cols, _ = csr
    gm = float(g['global_mean'])
    scale = np.unique(g['train_rating'])
    lo, hi = float(scale[0]), float(scale[-1])
    res = []
    for un, it, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist()):
        if un in users and it in items:
            uu = users[un]
            pred = S.predict_rating(P, Q, Y, Bu, Bi, cols[rowptr[uu]:rowptr[uu + 1]], uu, items[it], gm)
            pred = hi if pred > hi else lo if pred < lo else round(pred, 3)
        else:
            pred = gm
            pred = hi if pred > hi else lo if pred < lo else round(pred, 3)
        res.append([un, it, r, pred])
    return [m.strip() for m in Measure.ratingMeasure(res)]


def check_epoch(tabs, g, e, exact):
    k = int(g['row_stride'])
    last = e == len(g['loss']) - 1
    for name, t in zip(TABLES, tabs):
        for got, ref in ((t[::k], g[name + '_rows_epoch'][e]),) + (((t, g[name + '_last']),) if last else ()):
            if exact:
                assert np.array_equal(got, ref), (name, e)
            else:
                np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * float(np.abs(ref).max()))


def test_oracle_reproduces_reference_bits(g, ids):
    """Three epochs of the literal loop in the recorded visiting orders: every table after every epoch, the losses,
    the learning rates and the MAE / RMSE lines, all equal to the reference's."""
    u0, i0, csr, users, items = ids
    tabs = list(S.initial_tables(g))
    P, Q, Y, Bu, Bi = tabs
    gm = float(g['global_mean'])
    lr = float(g['lrate'][0][0])
    last = 0.0
    for e in range(len(g['loss'])):
        o = g['order_epoch'][e].astype(np.int64)
        sq = S.svdpp_sgd_sequential(P, Q, Y, Bu, Bi, u0[o], i0[o], g['train_rating'][o], csr[0], csr[1], lr,
                                    REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'], gm)
        loss = S.epoch_loss(sq, P, Q, Y, Bu, Bi, REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'])
        assert loss == g['loss'][e]
        check_epoch(tabs, g, e, exact=True)
        assert rating_lines(g, tabs, csr, users, items) == g['epoch_measure'][e].tolist()
        before = lr
        if not abs(last - loss) < 1e-3:
            lr = O.update_learning_rate(lr, 1.0, e + 1, last, loss)
        assert (before, lr) == tuple(g['lrate'][e])
        last = loss
    assert g['measure'].tolist() == g['epoch_measure'][-1].tolist()


def test_epoch_order_is_the_mt19937_shuffle(g):
    n = g['order_epoch'].shape[1]
    assert np.array_equal(g['order_epoch'][0], np.arange(n))
    rng = O.make_rng(state625=g['mt_state_before'])
    order = list(range(n))
    for e in range(g['order_epoch'].shape[0]):
        assert order == g['order_epoch'][e].tolist()
        rng.shuffle(order)
        assert np.array_equal(O.rng_state(rng), g['mt_state_after_epoch'][e])


def _longest_first(rowptr):
    return np.argsort(-np.diff(rowptr), kind='stable').astype(np.int32)


def test_closed_form_with_one_user_in_flight_is_the_literal_loop(g, ids):
    """svdpp_usermajor (one user at a time) == svdpp_sgd_sequential over the same user-major entries, float64,
    on FilmTrust (users with a single item included)."""
    _, _, csr, _, _ = ids
    rowptr = csr[0]
    assert (np.diff(rowptr) == 1).any()
    order = _longest_first(rowptr)
    u, i, r = S.user_entries(*csr, order)
    a = list(S.initial_tables(g))
    b = [t.copy() for t in a]
    gm, lr = float(g['global_mean']), 0.02
    la = S.svdpp_sgd_sequential(*a, u, i, r, rowptr, csr[1], lr, REG['reg_u'], REG['reg_i'], REG['reg_b'],
                                REG['reg_y'], gm)
    lb = S.svdpp_usermajor(*b, *csr, order, lr, REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'], gm)
    for x, y in zip(a, b):
        np.testing.assert_allclose(y, x, rtol=1e-12, atol=1e-12)
    assert abs(la - lb) <= 1e-12 * la


def test_device_step_source_replays_golden_epochs(g, ids, host):
    """float64: the parity kernel's arithmetic (column sums, dot grouping, step) over the three golden epochs."""
    u0, i0, csr, _, _ = ids
    tabs = list(S.initial_tables(g))
    gm = float(g['global_mean'])
    for e in range(len(g['loss'])):
        o = g['order_epoch'][e].astype(np.int64)
        lr = float(g['lrate'][e][0])
        sq = host_ordered(host, tabs, u0[o], i0[o], g['train_rating'][o], csr, lr, gm)
        loss = S.epoch_loss(sq, *tabs, REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'])
        assert abs(loss - g['loss'][e]) <= 1e-10 * g['loss'][e]
        check_epoch(tabs, g, e, exact=False)


def test_device_step_source_f32_tracks_the_f32_oracle(g, ids, host):
    u0, i0, csr, _, _ = ids
    n = 8000
    a = [t.astype(np.float32) for t in S.initial_tables(g)]
    b = [t.copy() for t in a]
    gm = float(g['global_mean'])
    args = (u0[:n], i0[:n], g['train_rating'][:n])
    host_ordered(host, a, *args, csr, 0.02, gm)
    S.svdpp_sgd_sequential(*b, *args, csr[0], csr[1], 0.02, REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'], gm)
    for x, y in zip(a, b):
        np.testing.assert_allclose(x, y, rtol=2e-4, atol=2e-6)


def test_device_closed_form_source_tracks_the_oracle(g, ids, host):
    """fp32 closed form of the fast kernel with one user in flight against the float64 closed form."""
    _, _, csr, _, _ = ids
    order = _longest_first(csr[0])
    ref = list(S.initial_tables(g))
    got = [t.astype(np.float32) for t in ref]
    ref = [t.astype(np.float32).astype(np.float64) for t in ref]
    gm = float(g['global_mean'])
    lg = host_usermajor(host, got, csr, order, 0.02, gm)
    lr_ = S.svdpp_usermajor(*ref, *csr, order, 0.02, REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'], gm)
    for x, y in zip(got, ref):
        np.testing.assert_allclose(x, y, rtol=2e-4, atol=2e-5)
    assert abs(lg - lr_) <= 1e-4 * lr_


def test_users_in_flight_reads_stale_rows():
    """users_in_flight = k sums the deltas of k users read from one snapshot: equal to one at a time when the users
    share no item, different when they do."""
    rng = np.random.default_rng(4)
    nu, ni, d = 6, 30, 8
    rowptr = np.array([0, 5, 9, 9, 10, 14, 19], dtype=np.int64)
    cols = rng.permutation(ni)[:19].astype(np.int32)             # disjoint item sets
    vals = rng.integers(1, 9, 19) / 2.0
    base = [rng.random((nu, d)) / 3, rng.random((ni, d)) / 3, rng.random((ni, d)), rng.random(nu), rng.random(ni)]
    order = np.arange(nu, dtype=np.int32)
    runs = []
    for k in (1, 3, 6):
        t = [x.copy() for x in base]
        S.svdpp_usermajor(*t, rowptr, cols, vals, order, 0.05, 0.01, 0.02, 0.1, 0.03, 3.0, users_in_flight=k)
        runs.append(t)
    for t in runs[1:]:
        for x, y in zip(t, runs[0]):
            np.testing.assert_allclose(x, y, rtol=1e-13, atol=1e-14)
    cols2 = cols.copy()
    cols2[5] = cols2[0]                                          # users 0 and 1 now share an item
    a, b = [x.copy() for x in base], [x.copy() for x in base]
    S.svdpp_usermajor(*a, rowptr, cols2, vals, order, 0.05, 0.01, 0.02, 0.1, 0.03, 3.0, users_in_flight=1)
    S.svdpp_usermajor(*b, rowptr, cols2, vals, order, 0.05, 0.01, 0.02, 0.1, 0.03, 3.0, users_in_flight=2)
    assert not np.allclose(a[1], b[1], rtol=0, atol=1e-12)


def test_model_class_resolves():
    from qrec_b200.QRec import _model_class
    from qrec_b200.model.rating.SVDPlusPlus import SVDPlusPlus
    assert _model_class('SVDPlusPlus') is SVDPlusPlus


def _golden_model(g, conf_extra, tmp_path, monkeypatch):
    from qrec_b200.model.rating.SVDPlusPlus import SVDPlusPlus
    from qrec_b200.util.config import ModelConf
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + conf_extra)
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    return SVDPlusPlus(conf, train, test)


def test_dropin_life_cycle_with_oracle_kernel(g, tmp_path, monkeypatch, capsys):
    """The drop-in from the golden seeds with the ordered kernel replaced by the oracle on CPU tensors: tables,
    losses, learning rates, MT19937 states, the configuration printout and every measure line."""
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.iterativeRecommender import IterativeRecommender

    def ordered(P, Q, Y, Bu, Bi, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y, gm, loss):
        assert P.dtype == torch.float64
        loss += S.svdpp_sgd_sequential(P.numpy(), Q.numpy(), Y.numpy(), Bu.numpy(), Bi.numpy(), u.numpy(), i.numpy(),
                                       r.numpy(), rowptr.numpy(), cols.numpy(), lr, reg_u, reg_i, reg_b, reg_y, gm)
        return loss

    def sumsq(x, out):
        out += float((x.numpy() * x.numpy()).sum())
        return out

    monkeypatch.setattr(E, 'svdpp_sgd_ordered', ordered)
    monkeypatch.setattr(E, 'sumsq', sumsq)
    monkeypatch.setattr(IterativeRecommender, '_device', lambda self: torch.device('cpu'))
    model = _golden_model(g, '', tmp_path, monkeypatch)
    seen = []
    orig = type(model).isConverged

    def spy(self, epoch):
        lr0 = self.lRate
        r = orig(self, epoch)
        seen.append((self.loss, lr0, self.lRate, np.array(random.getstate()[1], dtype=np.uint32),
                     [m.strip() for m in self.measure]))
        return r
    monkeypatch.setattr(type(model), 'isConverged', spy)
    measure = model.execute()
    assert 'regY: 0.010' in capsys.readouterr().out
    for name in TABLES:
        np.testing.assert_allclose(getattr(model, name), g[name + '_last'], rtol=1e-12, atol=1e-14)
    assert len(seen) == len(g['loss'])
    for e, (loss, lr0, lr1, st, lines) in enumerate(seen):
        assert abs(loss - g['loss'][e]) <= 1e-12 * g['loss'][e]
        assert (lr0, lr1) == tuple(g['lrate'][e])
        assert np.array_equal(st, g['mt_state_after_epoch'][e])
        assert lines == g['epoch_measure'][e].tolist()
    assert [m.strip() for m in measure] == g['measure'].tolist()
