"""WRMF on the CPU: the numpy oracle (oracle/wrmf_oracle.py) and the device arithmetic SOURCE
(qrec_b200/csrc/als_step.cuh, through tests/host_shims/als_step_host.cpp) against the golden run of the unmodified
reference's WRMF on FilmTrust (tests/golden/wrmf_filmtrust.npz, oracle/gen_golden_wrmf.py), the rating CSRs WRMF
consumes, and the drop-in's life cycle with the two kernels replaced by the oracle."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import wrmf_oracle as W          # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'wrmf_filmtrust.npz')
REG = 1.0                                     # reg.lambda -u of the golden conf; WRMF uses it on both sides


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def csrs(g):
    return W.golden_csrs(g)


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libals_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'als_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    for name, fp in (('host_als_side_f64', C.POINTER(C.c_double)), ('host_als_side_f32', C.POINTER(C.c_float))):
        fn = getattr(lib, name)
        fn.restype = C.c_int32
        fn.argtypes = [fp, fp, C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int32), fp,
                       C.c_double, C.c_double, C.POINTER(C.c_double)]
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def host_side(host, X, Z, csr, lam, alpha=W.ALPHA, with_loss=False):
    rowptr, cols, vals = csr
    f64 = X.dtype == np.float64
    ft = C.c_double if f64 else C.c_float
    vals = np.ascontiguousarray(vals, dtype=X.dtype)
    loss = np.zeros(1)
    fn = host.host_als_side_f64 if f64 else host.host_als_side_f32
    failed = fn(_p(X, ft), _p(Z, ft), X.shape[1], X.shape[0], Z.shape[0], _p(rowptr, C.c_int64), _p(cols, C.c_int32),
                _p(vals, ft), lam, alpha, _p(loss, C.c_double) if with_loss else None)
    return float(loss[0]), failed


def assert_table(got, ref):
    # rtol 1e-10 on every element; elements near zero are cancellations, held to 1e-12 of the table's scale
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * float(np.abs(ref).max()))


def assert_epoch(X, Y, g, e):
    """Tables after epoch e: every row_stride-th row after each epoch, all rows after the last one."""
    k = int(g['row_stride'])
    assert_table(X[::k], g['X_rows_epoch'][e])
    assert_table(Y[::k], g['Y_rows_epoch'][e])
    if e == len(g['loss']) - 1:
        assert_table(X, g['X_last'])
        assert_table(Y, g['Y_last'])


def test_oracle_reproduces_golden_epochs(g, csrs):
    X, Y = W.initial_tables(g)
    for e in range(len(g['loss'])):
        loss = W.epoch(X, Y, csrs[0], csrs[1], REG)
        assert abs(loss - g['loss'][e]) <= 1e-10 * g['loss'][e]
        assert_epoch(X, Y, g, e)


def test_device_step_source_replays_golden_epochs(g, csrs, host):
    """float64: Gram, accumulation, Cholesky and substitutions of als_step.cuh, three epochs."""
    X, Y = W.initial_tables(g)
    for e in range(len(g['loss'])):
        loss, failed = host_side(host, X, Y, csrs[0], REG, with_loss=True)
        assert failed == 0
        _, failed = host_side(host, Y, X, csrs[1], REG)
        assert failed == 0
        assert abs(loss - g['loss'][e]) <= 1e-10 * g['loss'][e]
        assert_epoch(X, Y, g, e)


def test_device_step_source_f32_tables_track_the_golden_run(g, csrs, host):
    """fp32 tables (A and b stay float64): only the stored rows are rounded."""
    X, Y = (t.astype(np.float32) for t in W.initial_tables(g))
    host_side(host, X, Y, csrs[0], REG, with_loss=True)
    host_side(host, Y, X, csrs[1], REG)
    k = int(g['row_stride'])
    for got, ref in ((X[::k], g['X_rows_epoch'][0]), (Y[::k], g['Y_rows_epoch'][0])):
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4 * float(np.abs(ref).max()))


def test_indefinite_system_fails_the_row_and_leaves_it_unchanged(host):
    rng = np.random.default_rng(3)
    d = 6
    Z = rng.random((10, d))
    X = rng.random((3, d))
    before = X.copy()
    rowptr = np.array([0, 3, 3, 5], dtype=np.int64)
    cols = np.array([0, 4, 7, 1, 2], dtype=np.int32)
    vals = np.array([1.0, 2.0, 3.0, 1.0, 1.0])
    # lambda far below -(largest eigenvalue of Z^T Z + alpha * sum v z z^T): A is negative definite for every row
    _, failed = host_side(host, X, Z, (rowptr, cols, vals), -1e6)
    assert failed == 3
    assert np.array_equal(X, before)
    # a positive definite system solves: row 1 has no entries -> (G + lambda I) x = 0
    _, failed = host_side(host, X, Z, (rowptr, cols, vals), 1.0)
    assert failed == 0 and np.array_equal(X[1], np.zeros(d))
    ref = before.copy()
    W.solve_side(ref, Z, rowptr, cols, vals, 1.0)
    np.testing.assert_allclose(X, ref, rtol=1e-12, atol=1e-14)


def _conf(evaluation):
    from qrec_b200.util.config import ModelConf
    return ModelConf.from_string('ratings.setup=-columns 0 1 2\nevaluation.setup=%s\n' % evaluation)


@pytest.mark.parametrize('evaluation', ['-ap 0.2', '-ap 0.2 -b 2'])
def test_rating_csr_matches_the_dict_views(evaluation, tmp_path):
    """Duplicate (user, item) lines collapse to one entry with the last value, in first-appearance position;
    with -b the loader has already dropped the low ratings and binarized the rest."""
    from qrec_b200.data.rating import Rating
    from qrec_b200.util.io import FileIO
    lines = ['u1 i1 3', 'u1 i2 1', 'u2 i1 4', 'u1 i1 5', 'u3 i3 2', 'u2 i3 3', 'u2 i1 1.5', 'u3 i2 4']
    path = tmp_path / 'r.txt'
    path.write_text('\n'.join(lines) + '\n')
    conf = _conf(evaluation)
    ev = evaluation.split()
    train = FileIO.loadDataSet(conf, str(path), binarized='-b' in ev, threshold=float(ev[-1]) if '-b' in ev else 0)
    data = Rating(conf, train, [])
    for by, sets, names, ids, other in (('user', data.trainSet_u, data.id2user, data.user, data.item),
                                        ('item', data.trainSet_i, data.id2item, data.item, data.user)):
        rowptr, cols, vals = data.rating_csr(by)
        assert rowptr.dtype == np.int64 and cols.dtype == np.int32 and vals.dtype == np.float64
        assert len(rowptr) == len(ids) + 1 and rowptr[-1] == sum(len(sets[n]) for n in ids)
        for k in range(len(ids)):
            row = sets[names[k]]
            a, b = rowptr[k], rowptr[k + 1]
            assert cols[a:b].tolist() == [other[n] for n in row]
            assert vals[a:b].tolist() == [float(v) for v in row.values()]
    rp, cols, vals = data.rating_csr('user')
    if '-b' in ev:
        assert set(vals.tolist()) == {1.0}
        assert 'u1' in data.user and cols[rp[data.user['u1']]:rp[data.user['u1'] + 1]].tolist() == [data.item['i1']]
    else:
        u1 = data.user['u1']
        assert cols[rp[u1]:rp[u1 + 1]].tolist() == [data.item['i1'], data.item['i2']]
        assert vals[rp[u1]:rp[u1 + 1]].tolist() == [5.0, 1.0]
        u2 = data.user['u2']
        assert vals[rp[u2]:rp[u2 + 1]].tolist() == [1.5, 3.0]


def test_model_class_resolves():
    from qrec_b200.QRec import _model_class
    from qrec_b200.model.ranking.WRMF import WRMF
    assert _model_class('WRMF') is WRMF


def test_row_order_is_longest_first():
    from qrec_b200.engine import als_row_order
    order = als_row_order(np.array([0, 2, 2, 7, 8, 10], dtype=np.int64))
    assert order.dtype == np.int32 and order.tolist() == [2, 0, 4, 3, 1]


def test_dropin_life_cycle_with_oracle_kernels(g, tmp_path, monkeypatch):
    """The drop-in from the golden seeds with als_gram / als_solve_rows replaced by the oracle on CPU tensors:
    tables, losses, learning rates, the MT19937 state after every epoch and the final measure lines."""
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.iterativeRecommender import IterativeRecommender
    from qrec_b200.model.ranking.WRMF import WRMF
    from qrec_b200.util.config import ModelConf

    def gram(Z, G=None, workspace=None):
        G.copy_(Z.double().T @ Z.double())
        return G

    def solve(X, Z, G, rowptr, cols, vals, lam, alpha, row_order, loss=None, n_failed=None):
        x = X.numpy()
        got = W.solve_side(x, Z.numpy(), rowptr.numpy(), cols.numpy(), vals.numpy(), lam, alpha,
                           rows=row_order.numpy(), with_loss=loss is not None)
        if loss is not None:
            loss += got
        return X

    monkeypatch.setattr(E, 'als_gram', gram)
    monkeypatch.setattr(E, 'als_solve_rows', solve)
    monkeypatch.setattr(IterativeRecommender, '_device', lambda self: torch.device('cpu'))
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']))
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    model = WRMF(conf, train, test)
    seen = []
    orig = WRMF.isConverged

    def spy(self, epoch):
        seen.append((self.loss, self.lRate))
        r = orig(self, epoch)
        seen[-1] += (self.lRate, np.array(random.getstate()[1], dtype=np.uint32))
        return r
    monkeypatch.setattr(WRMF, 'isConverged', spy)
    measure = model.execute()
    assert_table(model.X, g['X_last'])
    assert_table(model.Y, g['Y_last'])
    for e, (loss, lr0, lr1, st) in enumerate(seen):
        assert abs(loss - g['loss'][e]) <= 1e-10 * g['loss'][e]
        assert (lr0, lr1) == tuple(g['lrate'][e])
        assert np.array_equal(st, g['mt_state_after_epoch'][e])
    for got, ref in zip(measure, g['measure'].tolist()):
        assert got.strip().split(':')[0] == ref.split(':')[0]
        if ':' in ref:
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-6
