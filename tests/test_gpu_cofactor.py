"""K12 (CoFactor) on the GPU: qrec_cooc_count / engine.sppmi_csr against scipy's B^T B with the reference's filters,
qrec_cofactor_item_sweep_* against the in-order oracle (oracle/cofactor_oracle.py), and the drop-in against the
golden run of the reference's CoFactor (tests/golden/cofactor_filmtrust.npz).  Needs a GPU."""
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import cofactor_oracle as CO     # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'cofactor_filmtrust.npz')
DS = [1, 7, 20, 64, 128]


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _item_csr(rng, n_users, n_items, density, empty=()):
    """Item-major CSR of distinct users per item; the items in `empty` have none."""
    rows = []
    for i in range(n_items):
        k = 0 if i in empty else int(rng.binomial(n_users, density))
        rows.append(np.sort(rng.choice(n_users, k, replace=False)) if k else np.zeros(0, dtype=np.int64))
    rowptr = np.zeros(n_items + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    users = np.concatenate(rows).astype(np.int32) if rowptr[-1] else np.zeros(0, dtype=np.int32)
    return rowptr, users


def _check_cooc(torch, E, rowptr, users, n_users, filt):
    got = [t.cpu().numpy() for t in E.cooc_count(_dev(torch, rowptr), _dev(torch, users), n_users, filt)]
    _, ref = CO.sppmi(rowptr, users, n_users, 5, filt)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    assert np.array_equal(got[2].astype(np.int64), ref[2])
    return len(got[1])


@pytest.mark.parametrize('filt', [0, 1, 2])
def test_cooc_count_matches_scipy_on_random_data(torch, E, filt):
    rng = np.random.default_rng(filt)
    rowptr, users = _item_csr(rng, 400, 600, 0.02, empty=(0, 17, 599))
    assert _check_cooc(torch, E, rowptr, users, 400, filt) > 0


def test_cooc_count_wider_than_one_tile_and_edge_shapes(torch, E):
    rng = np.random.default_rng(7)
    rowptr, users = _item_csr(rng, 3000, 20000, 0.002, empty=(5, 8191, 8192, 19999))   # three column tiles
    assert _check_cooc(torch, E, rowptr, users, 3000, 2) > 0
    # a single user who rated everything: every pair shares exactly one user
    n = 50
    rowptr1 = np.arange(n + 1, dtype=np.int64)
    users1 = np.zeros(n, dtype=np.int32)
    assert _check_cooc(torch, E, rowptr1, users1, 1, 0) == n * (n - 1)
    assert _check_cooc(torch, E, rowptr1, users1, 1, 1) == 0
    # no entries at all
    assert _check_cooc(torch, E, np.zeros(4, dtype=np.int64), np.zeros(0, dtype=np.int32), 3, 0) == 0
    with pytest.raises(E.QRecError):
        E.cooc_count(_dev(torch, rowptr1), _dev(torch, users1 + 1), 1, 0)


def test_sppmi_on_filmtrust_matches_the_golden(torch, E):
    g = np.load(GOLD)
    _, (irp, icol, _) = CO.golden_csrs(g)
    n_users = len(g['user_names'])
    assert _check_cooc(torch, E, irp, icol, n_users, 2) > 0
    rowptr, cols, vals = (t.cpu().numpy() for t in E.sppmi_csr(_dev(torch, irp), _dev(torch, icol), n_users, 5, 2))
    assert np.array_equal(rowptr, g['sppmi_rowptr']) and np.array_equal(cols, g['sppmi_cols'])
    assert (np.abs(vals - g['sppmi_vals']) / np.spacing(g['sppmi_vals'])).max() <= 4


def _sweep_problem(d, seed, n_users=300, n_items=250, chain=False):
    rng = np.random.default_rng(seed)
    irp, icol = _item_csr(rng, n_users, n_items, 0.03, empty=(3,))
    ival = rng.integers(1, 6, len(icol)).astype(np.float64)
    if chain:                                     # item k's contexts are k - 1 and k + 1
        ctx = [[c for c in (k - 1, k + 1) if 0 <= c < n_items] for k in range(n_items)]
    else:                                         # random symmetric contexts, some items without any
        M = np.triu(rng.random((n_items, n_items)) < 0.03, 1)
        M[:, :20] = M[:20, :] = False
        M = M | M.T
        ctx = [np.flatnonzero(M[k]).tolist() for k in range(n_items)]
    srp = np.zeros(n_items + 1, dtype=np.int64)
    np.cumsum([len(r) for r in ctx], out=srp[1:])
    scol = np.array(sum(ctx, []), dtype=np.int32)
    U = rng.random((n_items, n_items))
    U = np.triu(U) + np.triu(U, 1).T
    sval = np.array([U[k, c] for k in range(n_items) for c in ctx[k]])
    X = rng.random((n_users, d)) / 3
    Y, G = rng.random((n_items, d)) / 3, rng.random((n_items, d)) / 10
    w, c = rng.random(n_items) / 10, rng.random(n_items) / 10
    return [Y, G, w, c, X], (irp, icol, ival), (srp, scol, sval)


def _gpu_sweep(torch, E, tabs, item_csr, sppmi, dtype, reg=1.0, gamma=1.0, **kw):
    T = [_dev(torch, a.astype(dtype)) for a in tabs]
    XtX = E.als_gram(T[4])
    dcsr = (_dev(torch, item_csr[0]), _dev(torch, item_csr[1]), _dev(torch, item_csr[2].astype(dtype)))
    dsp = (_dev(torch, sppmi[0]), _dev(torch, sppmi[1]), _dev(torch, sppmi[2].astype(dtype)))
    E.cofactor_item_sweep(*T[:4], T[4], XtX, dcsr, dsp, reg, gamma, CO.ALPHA, **kw)
    return [t.cpu().numpy() for t in T[:4]]


def _oracle_sweep(tabs, item_csr, sppmi, dtype, reg=1.0, gamma=1.0, items=None):
    Y, G, w, c, X = (a.astype(dtype) for a in tabs)          # float32 tables round every stored value
    sp = (sppmi[0], sppmi[1], sppmi[2].astype(dtype).astype(np.float64))
    CO.item_sweep(Y, G, w, c, X, item_csr, sp, reg, gamma, items=items)
    return [Y, G, w, c]


def _close(got, ref, tol):
    for a, b in zip(got, ref):
        np.testing.assert_allclose(a.astype(np.float64), b.astype(np.float64), rtol=0,
                                   atol=tol * float(np.abs(b).max()))


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('d', DS)
def test_item_sweep_matches_oracle(torch, E, dtype, d):
    tabs, item_csr, sppmi = _sweep_problem(d, seed=d)
    got = _gpu_sweep(torch, E, tabs, item_csr, sppmi, dtype)
    ref = _oracle_sweep(tabs, item_csr, sppmi, dtype)
    _close(got, ref, 1e-10 if dtype == 'float64' else 1e-4)
    no_ctx = np.diff(sppmi[0]) == 0
    for got_t, init in zip(got[1:], tabs[1:4]):               # G, w, c keep their values on items without contexts
        assert np.array_equal(got_t[no_ctx], init.astype(dtype)[no_ctx])
    again = _gpu_sweep(torch, E, tabs, item_csr, sppmi, dtype)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))


def test_chain_sppmi_follows_gauss_seidel_not_jacobi(torch, E):
    tabs, item_csr, sppmi = _sweep_problem(20, seed=11, n_items=300, chain=True)
    got = _gpu_sweep(torch, E, tabs, item_csr, sppmi, 'float64')
    gs = _oracle_sweep(tabs, item_csr, sppmi, 'float64')
    _close(got, gs, 1e-10)
    # Jacobi: every item from the state before the sweep
    jac = [a.copy() for a in tabs[:4]]
    for i in range(len(jac[2])):
        one = _oracle_sweep(tabs, item_csr, sppmi, 'float64', items=[i])
        for t, o in zip(jac, one):
            t[i] = o[i]
    err = max(np.abs(a - b).max() / np.abs(b).max() for a, b in zip(jac, gs))
    assert err > 1e-3                                          # the two orders differ by far more than rounding


def test_item_sweep_reuses_stamps_across_sweeps(torch, E):
    tabs, item_csr, sppmi = _sweep_problem(7, seed=4)
    stamps = torch.zeros(len(tabs[2]), dtype=torch.int32, device='cuda')
    T = [_dev(torch, a) for a in tabs]
    XtX = E.als_gram(T[4])
    dcsr = tuple(_dev(torch, a) for a in item_csr)
    dsp = tuple(_dev(torch, a) for a in sppmi)
    ref = [a.copy() for a in tabs]
    for sweep in (1, 2, 3):
        E.cofactor_item_sweep(*T[:4], T[4], XtX, dcsr, dsp, 1.0, 1.0, CO.ALPHA, stamps=stamps, sweep=sweep)
        CO.item_sweep(*ref[:4], ref[4], item_csr, sppmi, 1.0, 1.0)
    assert int(stamps.min()) == int(stamps.max()) == 3
    _close([t.cpu().numpy() for t in T[:4]], ref[:4], 1e-9)
    with pytest.raises(E.QRecError):                          # stamps of another sweep
        E.cofactor_item_sweep(*T[:4], T[4], XtX, dcsr, dsp, 1.0, 1.0, CO.ALPHA, stamps=stamps, sweep=2)


def test_item_sweep_counts_indefinite_systems_and_keeps_rows(torch, E):
    tabs, item_csr, sppmi = _sweep_problem(20, seed=5)
    n_ctx = int((np.diff(sppmi[0]) > 0).sum())
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    got = _gpu_sweep(torch, E, tabs, item_csr, sppmi, 'float64', gamma=-1e9, n_failed=n_failed)
    assert int(n_failed.item()) == n_ctx and np.array_equal(got[1], tabs[1])
    n_failed.zero_()
    got = _gpu_sweep(torch, E, tabs, item_csr, sppmi, 'float64', reg=-1e12, gamma=-1e9, n_failed=n_failed)
    assert int(n_failed.item()) == len(tabs[2]) + n_ctx
    assert np.array_equal(got[0], tabs[0]) and np.array_equal(got[1], tabs[1])
    with pytest.raises(E.QRecError):
        _gpu_sweep(torch, E, tabs, item_csr, sppmi, 'float64', gamma=-1e9)
    with pytest.raises(E.QRecError):
        _gpu_sweep(torch, E, [tabs[0][:, :1]] + tabs[1:], item_csr, sppmi, 'float64')


def _golden_model(conf_extra, tmp_path, monkeypatch):
    from qrec_b200.model.ranking.CoFactor import CoFactor
    from qrec_b200.util.config import ModelConf
    g = np.load(GOLD)
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + conf_extra)
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    return g, CoFactor(conf, train, test)


def test_dropin_reproduces_reference_run(torch, tmp_path, monkeypatch):
    """Default engine (float64 tables) from the golden seeds: X, Y, G, w, c after three epochs, the epoch losses and
    the final measure lines."""
    g, model = _golden_model('', tmp_path, monkeypatch)
    losses = []
    orig_print = print

    def spy_print(*args, **kw):
        if args and args[0] == 'epoch:':
            losses.append(args[3])
        orig_print(*args, **kw)
    monkeypatch.setattr('builtins.print', spy_print)
    measure = model.execute()
    monkeypatch.setattr('builtins.print', orig_print)
    has = np.diff(g['sppmi_rowptr']) > 0
    for got, ref in ((model.X, g['X_last']), (model.Y, g['Y_last']), (model.G[has], g['G_last_ctx']),
                     (model.w, g['w_last']), (model.c, g['c_last'])):
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-8 * float(np.abs(ref).max()))
    assert len(losses) == len(g['loss'])
    for got, ref in zip(losses, g['loss']):
        assert abs(got - ref) <= 1e-9 * ref
    for got, ref in zip(measure, g['measure'].tolist()):
        assert got.strip().split(':')[0] == ref.split(':')[0]
        if ':' in ref:
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-6


def test_dropin_fast_mode_with_gpu_eval_lands_near_reference(torch, tmp_path, monkeypatch):
    g, model = _golden_model('engine=-mode fast -eval gpu\n', tmp_path, monkeypatch)
    measure = model.execute()
    got = {m.split(':')[0]: float(m.split(':')[1]) for m in measure if ':' in m}
    ref = {m.split(':')[0]: float(m.split(':')[1]) for m in g['measure'].tolist() if ':' in m}
    for k in ('Precision', 'Recall'):
        assert abs(got[k] - ref[k]) < 0.01
