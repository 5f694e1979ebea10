"""K13 (ExpoMF) on the GPU: qrec_expomf_solve_rows_f32 against the float64 oracle (oracle/expomf_oracle.py) and the
drop-in against the golden run of the reference's ExpoMF (tests/golden/expomf_filmtrust.npz).  Needs a GPU.

Both sides solve in float64 and round the stored rows and priors to float32.  On an H100 every row and prior of these
tests came out with the oracle's exact float32 bits: the float64 results differ only in the grouping of the sums, far
below a float32 rounding step.  A value that lands on a rounding boundary may still round the other way, so the
bounds allow two float32 steps of the table's largest entry (rows) or of the value (priors)."""
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import expomf_oracle as EO          # noqa: E402
from test_expomf_cpu import assert_measure, assert_tables   # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'expomf_filmtrust.npz')
DS = [1, 7, 20, 50, 64, 128]
ROW_TOL = 2.4e-7        # kernel vs oracle, of the table's largest entry (float32 rows)
MU_TOL = 2.4e-7         # relative, on the prior


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


def _csr(rng, n_rows, n_z, empty=(), long_rows=()):
    """Unsorted distinct columns per row: mostly short rows, some empty, some longer than several staged blocks."""
    rows = []
    for r in range(n_rows):
        k = 0 if r in empty else (min(n_z, 230) if r in long_rows else int(rng.integers(1, 12)))
        rows.append(rng.choice(n_z, k, replace=False))
    rowptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum([len(c) for c in rows], out=rowptr[1:])
    return rowptr, np.concatenate(rows).astype(np.int32)


def _problem(d, seed, n_rows=450, n_z=700, x_scale=0.5, z_scale=0.3):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((n_rows, d)) * x_scale).astype(np.float32)
    Z = (rng.standard_normal((n_z, d)) * z_scale).astype(np.float32)
    rowptr, cols = _csr(rng, n_rows, n_z, empty=(0, 5, n_rows - 1), long_rows=(3, 100))
    mu_z = rng.uniform(0.001, 0.3, n_z).astype(np.float32)
    mu_x = rng.uniform(0.001, 0.3, n_rows).astype(np.float32)
    return X, Z, rowptr, cols, mu_z, mu_x


def _gpu_half(torch, E, X, Z, rowptr, cols, mu, mu_by_row, prior=False, max_ctas=0, lam=EO.LAM, **kw):
    Xd = _dev(torch, X)
    mu_out = torch.full((X.shape[0],), -1.0, dtype=torch.float32, device='cuda') if prior else None
    order = _dev(torch, _order(rowptr))
    E.expomf_half_epoch(Xd, _dev(torch, Z), _dev(torch, rowptr), _dev(torch, cols), _dev(torch, mu), mu_by_row, lam,
                        EO.LAM_Y, order, mu_out=mu_out, max_ctas=max_ctas, **kw)
    return Xd.cpu().numpy(), None if mu_out is None else mu_out.cpu().numpy()


def _order(rowptr):
    from qrec_b200.engine import als_row_order
    return als_row_order(rowptr)


def _oracle_half(X, Z, rowptr, cols, mu, mu_by_row, prior=False):
    X = X.copy()
    assert EO.solve_side(X, Z, rowptr, cols, mu, mu_by_row) == 0
    return X, (EO.prior_rows(X, Z, rowptr, cols, mu).astype(np.float32) if prior else None)


def _close(got, ref, tol):
    np.testing.assert_allclose(got.astype(np.float64), ref.astype(np.float64), rtol=0,
                               atol=tol * float(np.abs(ref).max()))


def _err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max() / np.abs(ref).max())


@pytest.mark.parametrize('d', DS)
def test_half_epochs_match_oracle(torch, E, d):
    """The user half (mu by column) and the item half with the prior (mu by row), with empty rows, rows longer than
    several staged blocks, and more rows than CTAs; the result is the same bits on any grid."""
    X, Z, rowptr, cols, mu_z, mu_x = _problem(d, seed=d)
    got, _ = _gpu_half(torch, E, X, Z, rowptr, cols, mu_z, False)
    ref, _ = _oracle_half(X, Z, rowptr, cols, mu_z, False)
    print('d=%d user half err %.3g' % (d, _err(got, ref)))
    _close(got, ref, ROW_TOL)
    assert not got[[0, 5, len(X) - 1]].any()                         # rows without entries solve to 0
    got2, mo = _gpu_half(torch, E, X, Z, rowptr, cols, mu_x, True, prior=True)
    ref2, mref = _oracle_half(X, Z, rowptr, cols, mu_x, True, prior=True)
    print('d=%d item half err %.3g prior err %.3g' % (d, _err(got2, ref2), _err(mo, mref)))
    _close(got2, ref2, ROW_TOL)
    np.testing.assert_allclose(mo, mref, rtol=MU_TOL)
    small, mo_small = _gpu_half(torch, E, X, Z, rowptr, cols, mu_x, True, prior=True, max_ctas=7)
    assert np.array_equal(small, got2) and np.array_equal(mo_small, mo)


def test_golden_scale_disparity(torch, E):
    """|theta| ~ 50 against |beta| ~ 0.03, as the golden run ends: both halves and the prior."""
    X, Z, rowptr, cols, mu_z, mu_x = _problem(20, seed=21, n_rows=600, n_z=500, x_scale=0.01, z_scale=20.0)
    got, mo = _gpu_half(torch, E, X, Z, rowptr, cols, mu_x, True, prior=True)      # items (small) against users (large)
    ref, mref = _oracle_half(X, Z, rowptr, cols, mu_x, True, prior=True)
    print('disparity item half err %.3g prior err %.3g' % (_err(got, ref), _err(mo, mref)))
    _close(got, ref, ROW_TOL)
    np.testing.assert_allclose(mo, mref, rtol=MU_TOL)
    Zs = (Z * 1e-3).astype(np.float32)
    Xl = (X * 2e3).astype(np.float32)
    got, _ = _gpu_half(torch, E, Xl, Zs, rowptr, cols, np.full(len(Zs), 0.01, np.float32), False)
    ref, _ = _oracle_half(Xl, Zs, rowptr, cols, np.full(len(Zs), 0.01, np.float32), False)
    print('disparity user half err %.3g' % _err(got, ref))
    _close(got, ref, ROW_TOL)


def test_square_tables_index_mu_by_column_with_prior(torch, E):
    """U == I: the item half indexes mu by the other table's row (the reference's quirk) while the prior still uses
    mu[r]; mu_out is a buffer of its own, so no CTA reads a prior another one wrote."""
    X, Z, rowptr, cols, mu_z, _ = _problem(20, seed=8, n_rows=400, n_z=400)
    got, mo = _gpu_half(torch, E, X, Z, rowptr, cols, mu_z, False, prior=True)
    ref, _ = _oracle_half(X, Z, rowptr, cols, mu_z, False)
    mref = EO.prior_rows(ref, Z, rowptr, cols, mu_z).astype(np.float32)
    _close(got, ref, ROW_TOL)
    np.testing.assert_allclose(mo, mref, rtol=MU_TOL)
    by_row, _ = _gpu_half(torch, E, X, Z, rowptr, cols, mu_z, True)
    assert np.abs(by_row - got).max() > 1e-3 * np.abs(got).max()


def _golden_epochs(torch, E, g, n_epochs, max_ctas=0):
    theta, beta, mu = (_dev(torch, a) for a in EO.initial_state(g, 20))
    (urp, ucol), (irp, icol) = EO.golden_csrs(g)
    uo, io = _dev(torch, _order(urp)), _dev(torch, _order(irp))
    urp, ucol, irp, icol = (_dev(torch, a) for a in (urp, ucol, irp, icol))
    nxt = torch.empty_like(mu)
    for _ in range(n_epochs):
        E.expomf_half_epoch(theta, beta, urp, ucol, mu, False, EO.LAM, EO.LAM_Y, uo, max_ctas=max_ctas)
        E.expomf_half_epoch(beta, theta, irp, icol, mu, True, EO.LAM, EO.LAM_Y, io, mu_out=nxt, max_ctas=max_ctas)
        mu, nxt = nxt, mu
    return [t.cpu().numpy() for t in (theta, beta, mu)]


def test_golden_epochs_are_bitwise_reproducible_on_any_grid(torch, E):
    g = np.load(GOLD)
    a = _golden_epochs(torch, E, g, 3)
    b = _golden_epochs(torch, E, g, 3)
    c = _golden_epochs(torch, E, g, 3, max_ctas=5)
    for x, y, z in zip(a, b, c):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    assert_tables(*a, g, 2)


def test_indefinite_systems_fail_and_keep_rows(torch, E):
    X, Z, rowptr, cols, mu_z, mu_x = _problem(7, seed=2)
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    got, mo = _gpu_half(torch, E, X, Z, rowptr, cols, mu_x, True, prior=True, lam=-1e6, n_failed=n_failed)
    assert int(n_failed.item()) == len(X) and np.array_equal(got, X)
    np.testing.assert_allclose(mo, EO.prior_rows(X, Z, rowptr, cols, mu_x).astype(np.float32), rtol=MU_TOL)
    with pytest.raises(E.QRecError):
        _gpu_half(torch, E, X, Z, rowptr, cols, mu_x, True, lam=-1e6)


def test_bad_arguments_raise(torch, E):
    X, Z, rowptr, cols, mu_z, mu_x = _problem(7, seed=3, n_rows=50, n_z=60)
    Xd, Zd, rp, cl, mz, mx = (_dev(torch, a) for a in (X, Z, rowptr, cols, mu_z, mu_x))
    order = _dev(torch, _order(rowptr))
    half = E.expomf_half_epoch
    bad = [
        lambda: half(Xd.double(), Zd, rp, cl, mz, False, 1e-5, 1.0, order),                   # float64 table
        lambda: half(Xd, Zd[:, :3], rp, cl, mz, False, 1e-5, 1.0, order),                      # widths differ
        lambda: half(torch.zeros(50, 129, device='cuda'), torch.zeros(60, 129, device='cuda'), rp, cl, mz, False,
                     1e-5, 1.0, order),                                                        # d > 128
        lambda: half(Xd, Xd, rp, cl, mx, True, 1e-5, 1.0, order),                              # X is Z
        lambda: half(Xd, Zd, rp, cl, mx, False, 1e-5, 1.0, order),                             # mu by column: 60
        lambda: half(Xd, Zd, rp, cl, mz, True, 1e-5, 1.0, order),                              # mu by row: 50
        lambda: half(Xd, Zd, rp, cl, mx, True, 1e-5, 1.0, order, mu_out=mx),                   # mu_out is mu
        lambda: half(Xd, Zd, rp, cl, mz, False, 1e-5, 1.0, order, mu_out=torch.empty_like(mx)),  # prior needs mu[r]
        lambda: half(Xd, Zd, rp[:-1], cl, mz, False, 1e-5, 1.0, order),                        # rowptr length
        lambda: half(Xd, Zd, rp, cl[:-1], mz, False, 1e-5, 1.0, order),                        # rowptr end
        lambda: half(Xd, Zd, rp, cl + 60, mz, False, 1e-5, 1.0, order),                        # column out of range
        lambda: half(Xd, Zd, rp, cl, mz, False, 1e-5, 1.0, order + 1),                         # row out of range
        lambda: half(Xd, Zd, rp, cl.long(), mz, False, 1e-5, 1.0, order),                      # int64 columns
        lambda: half(Xd.cpu(), Zd.cpu(), rp.cpu(), cl.cpu(), mz.cpu(), False, 1e-5, 1.0, order.cpu()),   # CPU tensors
    ]
    for k, call in enumerate(bad):
        with pytest.raises(E.QRecError):
            call()
            pytest.fail('bad argument set %d was accepted' % k)
    assert np.array_equal(Xd.cpu().numpy(), X)


def _golden_model(conf_extra, tmp_path, monkeypatch):
    from qrec_b200.model.ranking.ExpoMF import ExpoMF
    from qrec_b200.util.config import ModelConf
    g = np.load(GOLD)
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + conf_extra)
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    return g, ExpoMF(conf, train, test)


def test_dropin_reproduces_reference_run(torch, tmp_path, monkeypatch):
    """theta, beta, mu after three epochs within the CPU oracle's bounds, and the final measure lines."""
    g, model = _golden_model('', tmp_path, monkeypatch)
    measure = model.execute()
    print('drop-in measure', [m.strip() for m in measure], 'golden', g['measure'].tolist())
    for name in ('theta', 'beta', 'mu'):
        print('drop-in %s err %.3g' % (name, _err(getattr(model, name), g[name + '_epoch'][-1])))
    assert_tables(model.theta, model.beta, model.mu, g, len(g['mu_epoch']) - 1)
    assert_measure(measure, g)


def test_gpu_eval_gives_the_host_top_n(torch, tmp_path, monkeypatch):
    g, model = _golden_model('engine=-eval gpu\n', tmp_path, monkeypatch)
    measure = model.execute()
    _, N = model._top_n_setting()
    batched = model._recommend_all_on_device(N)
    assert batched is not None and len(batched) > 0
    same = sum(1 for u, rec in batched.items() if [n for n, _ in rec] == [n for n, _ in model._recommend(u, N)])
    print('-eval gpu: %d of %d top-%d lists equal the host ones' % (same, len(batched), N))
    assert same == len(batched)
    assert_measure(measure, g)
