"""ExpoMF on the CPU: the float64 oracle (oracle/expomf_oracle.py) against the golden run of the unmodified reference's
ExpoMF on FilmTrust (tests/golden/expomf_filmtrust.npz, oracle/gen_golden_expomf.py), the device arithmetic SOURCE
(qrec_b200/csrc/expomf_step.cuh with als_step.cuh, through tests/host_shims/expomf_step_host.cpp) against the oracle,
and the drop-in's life cycle with the kernel replaced by the oracle.

The reference forms its posteriors and Grams in float32; the oracle does everything in float64 and rounds only the
stored rows.  Over three epochs from the golden seed the largest deviation seen is 4.9e-5 of the table's largest
entry on theta, 2.1e-5 on beta and 2.3e-7 on mu; the bounds below are about three times that."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import expomf_oracle as EO      # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'expomf_filmtrust.npz')
D = 20
TOL = dict(theta=1.5e-4, beta=6.5e-5, mu=7e-7)     # of each table's largest entry


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def csrs(g):
    return EO.golden_csrs(g)


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libexpomf_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'expomf_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    dp, fp, i32p = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32)
    lib.host_expomf_solve_row.restype = C.c_int32
    lib.host_expomf_solve_row.argtypes = [dp, fp, C.c_int, C.c_int64, i32p, C.c_int64, fp, C.c_int, C.c_double,
                                          C.c_double, C.c_double, dp]
    lib.host_expomf_prior.restype = C.c_double
    lib.host_expomf_prior.argtypes = [dp, fp, C.c_int, C.c_int64, i32p, C.c_int64, C.c_double, C.c_double, C.c_double,
                                      C.c_double]
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def host_row(host, x_old, Z, cols, mu, mu_by_row, lam=EO.LAM):
    """(ok, x) from the header source; mu: a scalar when mu_by_row, else one float32 prior per row of Z."""
    x_old = np.ascontiguousarray(x_old, dtype=np.float64)
    Z = np.ascontiguousarray(Z, dtype=np.float32)
    cols = np.ascontiguousarray(cols, dtype=np.int32)
    mu_arr = np.ascontiguousarray(np.zeros(1, np.float32) if mu_by_row else mu, dtype=np.float32)
    out = x_old.copy()
    ok = host.host_expomf_solve_row(_p(x_old, C.c_double), _p(Z, C.c_float), Z.shape[1], Z.shape[0],
                                    _p(cols, C.c_int32), len(cols), _p(mu_arr, C.c_float), int(mu_by_row),
                                    float(mu) if mu_by_row else 0.0, lam, EO.LAM_Y, _p(out, C.c_double))
    return ok, out


def host_prior(host, x, Z, cols, mu_r):
    x = np.ascontiguousarray(x, dtype=np.float64)
    Z = np.ascontiguousarray(Z, dtype=np.float32)
    cols = np.ascontiguousarray(cols, dtype=np.int32)
    return host.host_expomf_prior(_p(x, C.c_double), _p(Z, C.c_float), Z.shape[1], Z.shape[0], _p(cols, C.c_int32),
                                  len(cols), float(mu_r), EO.LAM_Y, EO.A_PRIOR, EO.B_PRIOR)


def assert_tables(theta, beta, mu, g, e):
    for name, got in (('theta', theta), ('beta', beta), ('mu', mu)):
        ref = g[name + '_epoch'][e].astype(np.float64)
        np.testing.assert_allclose(got.astype(np.float64), ref, rtol=0, atol=TOL[name] * float(np.abs(ref).max()))


def test_oracle_reproduces_golden_epochs(g, csrs):
    theta, beta, mu = EO.initial_state(g, D)
    assert theta.dtype == beta.dtype == mu.dtype == np.float32
    for e in range(len(g['mu_epoch'])):
        assert EO.epoch(theta, beta, mu, *csrs) == 0
        assert_tables(theta, beta, mu, g, e)
    # the golden run's scale disparity, which the GPU tests reproduce
    assert np.abs(g['theta_epoch'][-1]).max() > 30 and np.abs(g['beta_epoch'][-1]).max() < 0.1


def test_prior_from_rows_equals_prior_from_users(g, csrs):
    theta, beta, mu = EO.initial_state(g, D)
    EO.epoch(theta, beta, mu, *csrs)
    irp, icol = csrs[1]
    np.testing.assert_allclose(EO.prior_rows(beta, theta, irp, icol, mu), EO.prior(theta, beta, mu, csrs[0]),
                               rtol=1e-12)


def _row_cases(rng):
    """(x_old, Z, cols, mu, mu_by_row) covering empty rows, a row that rated every column, mu near 0 and near 1,
    mu by column, and the golden scale disparity."""
    n_z, d = 300, 20
    Z = (rng.standard_normal((n_z, d)) * 0.3).astype(np.float32)
    x = rng.standard_normal(d) * 0.5
    some = np.sort(rng.choice(n_z, 25, replace=False))
    mu_col = rng.uniform(0.001, 0.2, n_z).astype(np.float32)
    big = (rng.standard_normal((n_z, d)) * 50).astype(np.float32)
    return [
        (x, Z, some, 0.01, True),
        (x, Z, np.zeros(0, np.int64), 0.01, True),                  # no entries: x = 0
        (x, Z, np.arange(n_z), 0.01, True),                         # rated every column: A = 1 everywhere
        (x, Z, some, np.float32(1e-6), True),                       # mu near 0
        (x, Z, some, np.float32(1 - 1e-6), True),                   # mu near 1
        (x, Z, some, mu_col, False),                                # mu by column
        (x, Z, rng.permutation(some), mu_col, False),               # unsorted columns
        (x * 1e-3, big, some, 0.01, True),                          # a small row against a large table
    ]


def test_device_step_source_rows_equal_oracle(host):
    rng = np.random.default_rng(3)
    for x, Z, cols, mu, by_row in _row_cases(rng):
        ok, got = host_row(host, x, Z, cols, mu, by_row)
        ref = EO.solve_row(x, Z, cols, float(mu) if by_row else mu)
        assert ok == 1 and ref is not None
        if len(cols) == 0:
            assert not got.any() and not ref.any()
            continue
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12 * float(np.abs(ref).max()))
        if by_row:
            p_ref = EO.prior_rows(got[None], Z, np.array([0, len(cols)]), cols, np.array([mu]))[0]
            assert abs(host_prior(host, got, Z, cols, mu) - p_ref) <= 1e-12 * p_ref


def test_device_step_source_replays_golden_first_epoch_rows(g, csrs, host):
    """Every 50th user of the first user half from the golden initial state, as the header source solves it."""
    theta, beta, mu = EO.initial_state(g, D)
    urp, ucol = csrs[0]
    for r in range(0, theta.shape[0], 50):
        ok, got = host_row(host, theta[r], beta, ucol[urp[r]:urp[r + 1]], mu, False)
        ref = EO.solve_row(theta[r], beta, ucol[urp[r]:urp[r + 1]], mu)
        assert ok == 1
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12 * float(np.abs(ref).max()))


def test_indefinite_system_fails_and_leaves_row_unchanged(host):
    rng = np.random.default_rng(4)
    x, Z, cols, mu, _ = _row_cases(rng)[0]
    ok, got = host_row(host, x, Z, cols, mu, True, lam=-1e6)
    assert ok == 0 and np.array_equal(got, x)
    assert EO.solve_row(x, Z, cols, mu, lam=-1e6) is None
    X = np.tile(x.astype(np.float32), (3, 1))
    rowptr = np.array([0, len(cols), len(cols), 2 * len(cols)])
    X0 = X.copy()
    assert EO.solve_side(X, Z, rowptr, np.concatenate([cols, cols]), np.full(3, mu, np.float32), True,
                         lam=-1e6) == 3
    assert np.array_equal(X, X0)


def _reference_solve_batch(X, X_old, Y_dense, mu, lam):
    """ExpoMF.py's _solve_batch / a_row_batch / _solve restated with numpy for a dense binary Y (rows of X_old):
    the indexing of mu is chosen by `mu.size == X.shape[0]`."""
    S = X_old.astype(np.float64).dot(X.astype(np.float64).T)
    m = mu.astype(np.float64) if mu.size == X.shape[0] else mu.astype(np.float64)[:X_old.shape[0], None]
    p = np.sqrt(EO.LAM_Y / 2 / np.pi) * np.exp(-EO.LAM_Y * S ** 2 / 2)
    A = (p + EO.EPS) / (p + EO.EPS + (1 - m) / m)
    A[Y_dense.nonzero()] = 1.0
    out = np.empty(X_old.shape)
    X64 = X.astype(np.float64)
    for k in range(X_old.shape[0]):
        B = X64.T.dot(A[k][:, None] * X64) + lam * np.eye(X.shape[1])
        out[k] = np.linalg.solve(B, np.dot(Y_dense[k] * A[k], X64))
    return out


def test_square_case_indexes_mu_by_user_like_the_reference():
    """U == I: the reference's item half takes mu by column, i.e. by USER id; the oracle's default does the same."""
    rng = np.random.default_rng(6)
    n, d = 40, 6
    Y = (rng.random((n, n)) < 0.15).astype(np.float64)
    theta = (rng.standard_normal((n, d)) * 2).astype(np.float32)
    beta = (rng.standard_normal((n, d)) * 0.5).astype(np.float32)
    mu = rng.uniform(0.001, 0.5, n).astype(np.float32)
    yt = Y.T
    irp = np.concatenate([[0], np.cumsum((yt > 0).sum(1))]).astype(np.int64)
    icol = np.concatenate([np.flatnonzero(row) for row in yt]).astype(np.int32)
    ref = _reference_solve_batch(theta, beta, yt, mu, EO.LAM)          # items against theta
    quirk, by_item = beta.copy(), beta.copy()
    EO.solve_side(quirk, theta, irp, icol, mu, False)                  # what epoch() picks when U == I
    EO.solve_side(by_item, theta, irp, icol, mu, True)
    np.testing.assert_allclose(quirk, ref.astype(np.float32), rtol=0, atol=1e-5 * np.abs(ref).max())
    assert np.abs(by_item - ref).max() > 1e-2 * np.abs(ref).max()     # the other indexing is visibly different
    # and epoch() itself takes the quirk when the tables have as many rows
    t2, b2, m2 = theta.copy(), beta.copy(), mu.copy()
    t3, b3, m3 = theta.copy(), beta.copy(), mu.copy()
    urp = np.concatenate([[0], np.cumsum((Y > 0).sum(1))]).astype(np.int64)
    ucol = np.concatenate([np.flatnonzero(row) for row in Y]).astype(np.int32)
    EO.epoch(t2, b2, m2, (urp, ucol), (irp, icol))
    EO.epoch(t3, b3, m3, (urp, ucol), (irp, icol), mu_by_row=False)
    assert np.array_equal(b2, b3) and np.array_equal(m2, m3)


def test_model_class_resolves():
    from qrec_b200.QRec import _model_class
    from qrec_b200.model.ranking.ExpoMF import ExpoMF
    assert _model_class('ExpoMF') is ExpoMF


def oracle_half_epoch(X, Z, rowptr, cols, mu, mu_by_row, lam, lam_y, row_order, mu_out=None, a=1.0, b=99.0,
                      n_failed=None, max_ctas=0):
    """engine.expomf_half_epoch on CPU tensors through the oracle."""
    rows = row_order.numpy()
    if mu_out is not None:
        Xn = X.numpy()
        assert EO.solve_side(Xn, Z.numpy(), rowptr.numpy(), cols.numpy(), mu.numpy(), mu_by_row, lam, lam_y, rows) == 0
        mu_out.numpy()[rows] = EO.prior_rows(Xn, Z.numpy(), rowptr.numpy(), cols.numpy(), mu.numpy(), a, b, lam_y, rows)
    else:
        assert EO.solve_side(X.numpy(), Z.numpy(), rowptr.numpy(), cols.numpy(), mu.numpy(), mu_by_row, lam, lam_y,
                             rows) == 0
    return X


def test_dropin_life_cycle_with_oracle_kernel(g, tmp_path, monkeypatch):
    """The drop-in from the golden seed with expomf_half_epoch replaced by the oracle on CPU tensors: the initModel
    draws, the printed lines, the tables after the last epoch and the ranking."""
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.iterativeRecommender import IterativeRecommender
    from qrec_b200.model.ranking.ExpoMF import ExpoMF
    from qrec_b200.util.config import ModelConf

    calls = []

    def half(*args, **kw):
        calls.append((args[5], kw.get('mu_out') is not None))
        return oracle_half_epoch(*args, **kw)

    monkeypatch.setattr(E, 'expomf_half_epoch', half)
    monkeypatch.setattr(IterativeRecommender, '_device', lambda self: torch.device('cpu'))
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']))
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    model = ExpoMF(conf, train, test)
    lines, mus = [], []
    orig_print = print

    def spy_print(*args, **kw):
        if args and isinstance(args[0], str):
            lines.append(args[0])
        elif args and isinstance(args[0], np.ndarray):
            mus.append(args[0].copy())
        orig_print(*args, **kw)
    monkeypatch.setattr('builtins.print', spy_print)
    measure = model.execute()
    monkeypatch.undo()
    n_epochs = len(g['mu_epoch'])
    theta0, beta0, mu0 = EO.initial_state(g, D)
    assert calls == [(False, False), (True, True)] * n_epochs          # FilmTrust has more items than users
    epoch_lines = [s for s in lines if s.startswith('epoch #') or s == '\tUpdating exposure prior...']
    assert epoch_lines == sum((['epoch #%d' % e, '\tUpdating exposure prior...'] for e in range(n_epochs)), [])
    assert len(mus) == n_epochs and np.array_equal(mus[0], mu0)          # each epoch prints the mu it started from
    for e in range(1, n_epochs):
        np.testing.assert_allclose(mus[e], g['mu_epoch'][e - 1], rtol=0, atol=TOL['mu'] * g['mu_epoch'][e - 1].max())
    assert model.theta.dtype == model.beta.dtype == model.mu.dtype == np.float32
    assert_tables(model.theta, model.beta, model.mu, g, n_epochs - 1)
    u = g['test_users'][0]
    assert np.array_equal(model.predictForRanking(u), model.beta.dot(model.theta[model.data.getUserId(u)]))
    assert_measure(measure, g)


def assert_measure(measure, g):
    """Precision, recall and F1 to the printed digits; NDCG within 3e-5 -- the float64 tables swap one pair of
    neighbours inside a top-10 list against the reference's float32 ones (NDCG off by 1.1e-5)."""
    assert len(measure) == len(g['measure'])
    for got, ref in zip(measure, g['measure'].tolist()):
        if ref.startswith('NDCG:'):
            assert got.startswith('NDCG:') and abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 3e-5
        else:
            assert got.strip() == ref
