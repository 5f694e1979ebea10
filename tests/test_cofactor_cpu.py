"""CoFactor on the CPU: the numpy oracle (oracle/cofactor_oracle.py) and the device arithmetic SOURCE
(qrec_b200/csrc/cofactor_step.cuh with als_step.cuh, through tests/host_shims/cofactor_step_host.cpp) against the
golden run of the unmodified reference's CoFactor on FilmTrust (tests/golden/cofactor_filmtrust.npz,
oracle/gen_golden_cofactor.py), and the drop-in's life cycle with the kernels replaced by the oracle.

Tolerances come from the observed oracle-vs-golden error.  The oracle and the shim sum in other orders than the
reference and solve instead of inverting; over three epochs their largest deviation from the golden tables is
5e-11 of the table's largest entry (G, whose systems sum_c Y_c Y_c^T + 0.01 I often have fewer contexts than d and
are far worse conditioned than WRMF's), and 1e-14 relative on the losses.  Tables are held to 1e-9 of their scale,
losses to 1e-12 relative.  The SPPMI matches exactly (same sparsity pattern; values within 4 ulp)."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import cofactor_oracle as CO      # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'cofactor_filmtrust.npz')
REG, GAMMA, K, FILTER, D = 1.0, 0.01, 5, 2, 20     # the golden conf: reg.lambda -u 1, CoFactor=-k 5 -gamma 0.01 -filter 2


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def csrs(g):
    return CO.golden_csrs(g)


@pytest.fixture(scope='module')
def sppmi(g):
    return g['sppmi_rowptr'], g['sppmi_cols'], g['sppmi_vals']


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libcofactor_step_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'cofactor_step_host.cpp'), '-o', out])
    lib = C.CDLL(out)
    fn = lib.host_cofactor_item_sweep_f64
    dp, i64p, i32p = C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_int32)
    fn.restype = C.c_int32
    fn.argtypes = [dp, dp, dp, dp, dp, C.c_int, C.c_int64, C.c_int64, i64p, i32p, dp, i64p, i32p, dp,
                   C.c_double, C.c_double, C.c_double]
    return lib


def host_item_sweep(host, Y, G, w, c, X, item_csr, sppmi, reg=REG, gamma=GAMMA):
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))                 # noqa: E731
    irp, icol, ival = (np.ascontiguousarray(a) for a in item_csr)
    srp, scol, sval = (np.ascontiguousarray(a) for a in sppmi)
    dd = C.c_double
    return host.host_cofactor_item_sweep_f64(p(Y, dd), p(G, dd), p(w, dd), p(c, dd), p(X, dd), X.shape[1], X.shape[0],
                                             Y.shape[0], p(irp, C.c_int64), p(icol, C.c_int32), p(ival, dd),
                                             p(srp, C.c_int64), p(scol, C.c_int32), p(sval, dd), reg, gamma, CO.ALPHA)


def assert_table(got, ref):
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-9 * float(np.abs(ref).max()))


def assert_epoch(X, Y, G, w, c, g, e):
    """Y, G every row_stride-th row after each epoch; everything after the last one (G: the rows with contexts)."""
    k = int(g['row_stride'])
    assert_table(Y[::k], g['Y_rows_epoch'][e])
    assert_table(G[::k], g['G_rows_epoch'][e])
    if e == len(g['loss']) - 1:
        has = np.diff(g['sppmi_rowptr']) > 0
        for got, ref in ((X, g['X_last']), (Y, g['Y_last']), (G[has], g['G_last_ctx']), (w, g['w_last']),
                         (c, g['c_last'])):
            assert_table(got, ref)


def test_oracle_sppmi_matches_golden(g, csrs):
    (rowptr, cols, vals), _ = CO.sppmi(*csrs[1][:2], len(g['user_names']), K, FILTER)
    assert np.array_equal(rowptr, g['sppmi_rowptr']) and np.array_equal(cols, g['sppmi_cols'])
    ulp = np.abs(vals - g['sppmi_vals']) / np.spacing(g['sppmi_vals'])
    assert ulp.max() <= 4
    # symmetric, as the item sweep's ordering argument needs
    n = len(rowptr) - 1
    rows = np.repeat(np.arange(n), np.diff(rowptr))
    assert set(zip(rows.tolist(), cols.tolist())) == set(zip(cols.tolist(), rows.tolist()))


def test_oracle_reproduces_golden_epochs(g, csrs, sppmi):
    X, Y, w, c, G = CO.initial_state(g, D)
    for e in range(len(g['loss'])):
        loss = CO.epoch(X, Y, G, w, c, csrs[0], csrs[1], sppmi, REG, GAMMA)
        assert abs(loss - g['loss'][e]) <= 1e-12 * g['loss'][e]
        assert_epoch(X, Y, G, w, c, g, e)


def test_device_step_source_replays_golden_item_sweeps(g, csrs, sppmi, host):
    """The user side from the oracle (WRMF's, pinned by test_wrmf_cpu.py), the item sweep from the header source."""
    X, Y, w, c, G = CO.initial_state(g, D)
    from oracle import wrmf_oracle as W
    for e in range(len(g['loss'])):
        W.solve_side(X, Y, *csrs[0], REG, with_loss=True)
        assert host_item_sweep(host, Y, G, w, c, X, csrs[1], sppmi) == 0
        assert_epoch(X, Y, G, w, c, g, e)


def test_device_step_source_indefinite_systems_leave_rows_unchanged(g, csrs, sppmi, host):
    X, Y, w, c, G = CO.initial_state(g, D)
    Y0, G0 = Y.copy(), G.copy()
    n_items = Y.shape[0]
    n_ctx = int((np.diff(g['sppmi_rowptr']) > 0).sum())
    # gamma far below -(largest eigenvalue of sum Y_c Y_c^T): every G system is negative definite; Y's are fine
    failed = host_item_sweep(host, Y, G, w, c, X, csrs[1], sppmi, gamma=-1e9)
    assert failed == n_ctx and np.array_equal(G, G0) and not np.array_equal(Y, Y0)
    # regU far below: every Y system fails too
    X, Y, w, c, G = CO.initial_state(g, D)
    failed = host_item_sweep(host, Y, G, w, c, X, csrs[1], sppmi, reg=-1e12, gamma=-1e9)
    assert failed == n_items + n_ctx and np.array_equal(Y, Y0) and np.array_equal(G, G0)


def test_model_class_resolves():
    from qrec_b200.QRec import _model_class
    from qrec_b200.model.ranking.CoFactor import CoFactor
    assert _model_class('CoFactor') is CoFactor


def test_gauss_seidel_depth_of_a_chain_and_the_golden():
    n = 9
    rowptr = np.zeros(n + 1, dtype=np.int64)
    rows = [[k for k in (i - 1, i + 1) if 0 <= k < n] for i in range(n)]
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    assert CO.gauss_seidel_depth(rowptr, np.array(sum(rows, []), dtype=np.int32)) == n


def test_dropin_life_cycle_with_oracle_kernels(g, tmp_path, monkeypatch):
    """The drop-in from the golden seeds with sppmi_csr / als_gram / als_solve_rows / cofactor_item_sweep replaced
    by the oracle on CPU tensors: tables, w, c, losses and the final measure lines."""
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.iterativeRecommender import IterativeRecommender
    from qrec_b200.model.ranking.CoFactor import CoFactor
    from qrec_b200.util.config import ModelConf
    from oracle import wrmf_oracle as W

    def sppmi_csr(rowptr, cols, num_users, k, filt, dtype=None):
        (rp, cl, vl), _ = CO.sppmi(rowptr.numpy(), cols.numpy(), num_users, k, filt)
        return torch.from_numpy(rp), torch.from_numpy(cl), torch.from_numpy(vl)

    def gram(Z, G=None, workspace=None):
        G.copy_(Z.double().T @ Z.double())
        return G

    def solve(X, Z, G, rowptr, cols, vals, lam, alpha, row_order, loss=None, n_failed=None):
        got = W.solve_side(X.numpy(), Z.numpy(), rowptr.numpy(), cols.numpy(), vals.numpy(), lam, alpha,
                           rows=row_order.numpy(), with_loss=loss is not None)
        if loss is not None:
            loss += got
        return X

    sweeps = []

    def item_sweep(Y, G, w, c, X, XtX, item_csr, sppmi, lam, gamma, alpha, n_failed=None, stamps=None, sweep=1):
        sweeps.append(sweep)
        CO.item_sweep(Y.numpy(), G.numpy(), w.numpy(), c.numpy(), X.numpy(), [a.numpy() for a in item_csr],
                      [a.numpy() for a in sppmi], lam, gamma, alpha)
        return Y

    monkeypatch.setattr(E, 'sppmi_csr', sppmi_csr)
    monkeypatch.setattr(E, 'als_gram', gram)
    monkeypatch.setattr(E, 'als_solve_rows', solve)
    monkeypatch.setattr(E, 'cofactor_item_sweep', item_sweep)
    monkeypatch.setattr(IterativeRecommender, '_device', lambda self: torch.device('cpu'))
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']))
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    model = CoFactor(conf, train, test)
    losses = []
    orig_print = print

    def spy_print(*args, **kw):
        if args and args[0] == 'epoch:':
            losses.append(args[3])
        orig_print(*args, **kw)
    monkeypatch.setattr('builtins.print', spy_print)
    measure = model.execute()
    monkeypatch.undo()
    assert (model.negCount, model.regR, model.filter) == (K, GAMMA, FILTER)
    assert sweeps == [1, 2, 3]
    assert_epoch(model.X, model.Y, model.G, model.w, model.c, g, len(g['loss']) - 1)
    assert len(losses) == len(g['loss'])
    for got, ref in zip(losses, g['loss']):
        assert abs(got - ref) <= 1e-12 * ref
    for got, ref in zip(measure, g['measure'].tolist()):
        assert got.strip().split(':')[0] == ref.split(':')[0]
        if ':' in ref:
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-6
