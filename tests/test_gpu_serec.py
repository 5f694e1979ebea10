"""K14 (SERec) on the GPU: qrec_serec_solve_rows_f32 against the float64 oracle (oracle/serec_oracle.py, the prior as a
single product deg * A, as the kernel forms it) and the drop-in against the golden run of the reference's SERec
(tests/golden/serec_filmtrust.npz).  Needs a GPU.

Both sides solve in float64 and round the stored rows to float32; the float64 results differ only in the grouping of
the sums, far below a float32 rounding step, but a value that lands on a rounding boundary may still round the other
way, so the bounds allow two float32 steps of the table's largest entry.  The summed posteriors are float64 on both
sides: they are checked against the oracle's sums over the kernel's own new rows, to 1e-12 relative."""
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import expomf_oracle as EO          # noqa: E402
from oracle import serec_oracle as SO           # noqa: E402
from test_serec_cpu import TOL, assert_measure, relation   # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'serec_filmtrust.npz')
DS = [1, 7, 20, 50, 64, 128]
ROW_TOL = 2.4e-7        # kernel vs oracle, of the table's largest entry (float32 rows)
ASUM_TOL = 1e-12        # relative, on the summed posteriors


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


def _order(rowptr):
    from qrec_b200.engine import als_row_order
    return als_row_order(rowptr)


def _problem(d, seed, nu=450, ni=700):
    """theta [nu], beta [ni], the user- and item-major CSRs (unsorted columns; users 0, 5 and the last without
    entries, users 3 and 100 with more than several staged blocks), degrees with zeros, ones and a long tail, and
    summed posteriors A in (0.5, 0.3 U)."""
    rng = np.random.default_rng(seed)
    theta = (rng.standard_normal((nu, d)) * 0.5).astype(np.float32)
    beta = (rng.standard_normal((ni, d)) * 0.3).astype(np.float32)
    rows = []
    for u in range(nu):
        k = 0 if u in (0, 5, nu - 1) else (min(ni, 230) if u in (3, 100) else int(rng.integers(1, 12)))
        rows.append(rng.choice(ni, k, replace=False))
    urp = np.zeros(nu + 1, dtype=np.int64)
    np.cumsum([len(c) for c in rows], out=urp[1:])
    ucol = np.concatenate(rows).astype(np.int32)
    users = np.repeat(np.arange(nu), np.diff(urp))
    order = np.argsort(ucol, kind='stable')
    irp = np.zeros(ni + 1, dtype=np.int64)
    np.cumsum(np.bincount(ucol, minlength=ni), out=irp[1:])
    icol = users[order].astype(np.int32)
    deg = np.where(rng.random(nu) < 0.5, 0, np.minimum(rng.zipf(1.6, nu), 3000)).astype(np.int32)
    deg[1], deg[2] = 1, 3000
    A = rng.uniform(0.5, 0.3 * nu, ni)
    return theta, beta, (urp, ucol), (irp, icol), deg, A


def _priors(A, deg, row_is_user, n, m):
    """(solve prior [n, m], fused-pass prior [n, m]) of a half-epoch over n rows against m."""
    U = n if row_is_user else m
    if A is None:
        M = np.full((n, m), SO.MU0)
        return M, M
    P = SO.prior(A, deg, U)
    return (P if row_is_user else P.T), (P.T if len(A) == n and len(deg) == m else None)


def _gpu_half(torch, E, X, Z, csr, A, deg, row_is_user, out=False, max_ctas=0, lam=SO.LAM, **kw):
    Xd = _dev(torch, X)
    asum_out = torch.full((X.shape[0],), -1.0, dtype=torch.float64, device='cuda') if out else None
    E.serec_half_epoch(Xd, _dev(torch, Z), _dev(torch, csr[0]), _dev(torch, csr[1]),
                       None if A is None else _dev(torch, A), _dev(torch, deg), row_is_user, lam, SO.LAM_Y,
                       _dev(torch, _order(csr[0])), asum_out=asum_out, max_ctas=max_ctas, **kw)
    return Xd.cpu().numpy(), None if asum_out is None else asum_out.cpu().numpy()


def _oracle_half(X, Z, csr, A, deg, row_is_user):
    M, _ = _priors(A, deg, row_is_user, len(X), len(Z))
    X = X.copy()
    assert SO.solve_side(X, Z, csr[0], csr[1], M) == 0
    return X


def _oracle_asum(X_new, Z, csr, A, deg, row_is_user):
    _, Mo = _priors(A, deg, row_is_user, len(X_new), len(Z))
    return SO.asum_rows(X_new, Z, csr[0], csr[1], Mo)


def _close(got, ref, tol):
    np.testing.assert_allclose(got.astype(np.float64), ref.astype(np.float64), rtol=0,
                               atol=tol * float(np.abs(ref).max()))


def _err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max() / np.abs(ref).max())


@pytest.mark.parametrize('d', DS)
def test_half_epochs_match_oracle(torch, E, d):
    """Both halves in both prior modes (social from A and deg, uniform mu0), users of degree 0 to 3000, empty and long
    rows, more rows than CTAs; the item half with and without the fused sums, on any grid, gives the same bits."""
    theta, beta, ucsr, icsr, deg, A = _problem(d, seed=d)
    for mode, Am in (('social', A), ('uniform', None)):
        got, _ = _gpu_half(torch, E, theta, beta, ucsr, Am, deg, True)
        ref = _oracle_half(theta, beta, ucsr, Am, deg, True)
        print('d=%d %s user half err %.3g' % (d, mode, _err(got, ref)))
        _close(got, ref, ROW_TOL)
        assert not got[[0, 5, len(theta) - 1]].any()                    # users without entries solve to 0
        got2, asum = _gpu_half(torch, E, beta, theta, icsr, Am, deg, False, out=True)
        ref2 = _oracle_half(beta, theta, icsr, Am, deg, False)
        aref = _oracle_asum(got2, theta, icsr, Am, deg, False)
        print('d=%d %s item half err %.3g asum err %.3g' % (d, mode, _err(got2, ref2), _err(asum, aref)))
        _close(got2, ref2, ROW_TOL)
        np.testing.assert_allclose(asum, aref, rtol=ASUM_TOL)
        plain, none = _gpu_half(torch, E, beta, theta, icsr, Am, deg, False)
        small, asum_small = _gpu_half(torch, E, beta, theta, icsr, Am, deg, False, out=True, max_ctas=7)
        assert none is None and np.array_equal(plain, got2)
        assert np.array_equal(small, got2) and np.array_equal(asum_small, asum)


def test_the_prior_depends_on_the_degree(torch, E):
    """The same user with degree 0 and with a high degree solves to visibly different rows; with A absent the degree
    does not matter."""
    theta, beta, ucsr, _, deg, A = _problem(20, seed=4)
    low, high = deg.copy(), deg.copy()
    low[:], high[:] = 0, 40
    a, _ = _gpu_half(torch, E, theta, beta, ucsr, A, low, True)
    b, _ = _gpu_half(torch, E, theta, beta, ucsr, A, high, True)
    assert np.abs(a - b).max() > 1e-3 * np.abs(a).max()
    _close(b, _oracle_half(theta, beta, ucsr, A, high, True), ROW_TOL)
    u0, _ = _gpu_half(torch, E, theta, beta, ucsr, None, low, True)
    u1, _ = _gpu_half(torch, E, theta, beta, ucsr, None, high, True)
    assert np.array_equal(u0, u1)


def test_square_tables_take_the_user_branch_with_fused_sums(torch, E):
    """U == I: the item half reads mu[i, u] (the reference's quirk: row_is_user for item rows) while the fused sums
    still read mu[u, i]; asum_out is a buffer of its own, so no CTA reads a sum another one wrote."""
    theta, beta, ucsr, icsr, deg, A = _problem(20, seed=8, nu=400, ni=400)
    got, asum = _gpu_half(torch, E, beta, theta, icsr, A, deg, True, out=True)
    P = SO.prior(A, deg, 400)
    ref = beta.copy()
    assert SO.solve_side(ref, theta, icsr[0], icsr[1], P) == 0
    _close(got, ref, ROW_TOL)
    np.testing.assert_allclose(asum, SO.asum_rows(got, theta, icsr[0], icsr[1], P.T), rtol=ASUM_TOL)
    by_item, _ = _gpu_half(torch, E, beta, theta, icsr, A, deg, False)
    assert np.abs(by_item - got).max() > 1e-3 * np.abs(got).max()


def _golden_epochs(torch, E, g, n_epochs, max_ctas=0):
    theta, beta = (_dev(torch, a) for a in SO.initial_state(g, 20))
    (urp, ucol), (irp, icol) = EO.golden_csrs(g)
    uo, io = _dev(torch, _order(urp)), _dev(torch, _order(irp))
    urp, ucol, irp, icol, deg = (_dev(torch, a) for a in (urp, ucol, irp, icol, g['deg']))
    asum, nxt = None, torch.empty(len(g['item_names']), dtype=torch.float64, device='cuda')
    for _ in range(n_epochs):
        E.serec_half_epoch(theta, beta, urp, ucol, asum, deg, True, SO.LAM, SO.LAM_Y, uo, max_ctas=max_ctas)
        E.serec_half_epoch(beta, theta, irp, icol, asum, deg, False, SO.LAM, SO.LAM_Y, io, asum_out=nxt,
                           max_ctas=max_ctas)
        asum, nxt = nxt, (torch.empty_like(nxt) if asum is None else asum)
    return [t.cpu().numpy() for t in (theta, beta, asum)]


def _assert_golden(theta, beta, asum, g, e):
    for name, got in (('theta', theta), ('beta', beta), ('asum', asum)):
        ref = g[name + '_epoch'][e].astype(np.float64)
        print('%s err %.3g' % (name, _err(got, ref)))
        np.testing.assert_allclose(got.astype(np.float64), ref, rtol=0, atol=TOL[name] * float(np.abs(ref).max()))


def test_golden_epochs_are_bitwise_reproducible_on_any_grid(torch, E):
    g = np.load(GOLD)
    a = _golden_epochs(torch, E, g, 3)
    b = _golden_epochs(torch, E, g, 3)
    c = _golden_epochs(torch, E, g, 3, max_ctas=5)
    for x, y, z in zip(a, b, c):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    _assert_golden(*a, g, 2)


def test_indefinite_systems_fail_and_keep_rows(torch, E):
    theta, beta, _, icsr, deg, A = _problem(7, seed=2)
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    got, asum = _gpu_half(torch, E, beta, theta, icsr, A, deg, False, out=True, lam=-1e6, n_failed=n_failed)
    assert int(n_failed.item()) == len(beta) and np.array_equal(got, beta)
    np.testing.assert_allclose(asum, _oracle_asum(beta, theta, icsr, A, deg, False), rtol=ASUM_TOL)
    with pytest.raises(E.QRecError):
        _gpu_half(torch, E, beta, theta, icsr, A, deg, False, lam=-1e6)


def test_bad_arguments_raise(torch, E):
    theta, beta, ucsr, icsr, deg, A = _problem(7, seed=3, nu=50, ni=60)
    Xd, Zd, rp, cl, dg, Ad = (_dev(torch, a) for a in (theta, beta, ucsr[0], ucsr[1], deg, A))
    order = _dev(torch, _order(ucsr[0]))
    irp, icl, iorder = _dev(torch, icsr[0]), _dev(torch, icsr[1]), _dev(torch, _order(icsr[0]))
    out = torch.empty(60, dtype=torch.float64, device='cuda')
    half = E.serec_half_epoch
    bad = [
        lambda: half(Xd.double(), Zd, rp, cl, Ad, dg, True, 1e-3, 0.01, order),                 # float64 table
        lambda: half(Xd, Zd[:, :3], rp, cl, Ad, dg, True, 1e-3, 0.01, order),                    # widths differ
        lambda: half(torch.zeros(50, 129, device='cuda'), torch.zeros(60, 129, device='cuda'), rp, cl, Ad, dg, True,
                     1e-3, 0.01, order),                                                         # d > 128
        lambda: half(Xd, Xd, rp, cl, Ad, dg, True, 1e-3, 0.01, order),                           # X is Z
        lambda: half(Xd, Zd, rp, cl, Ad.float(), dg, True, 1e-3, 0.01, order),                   # float32 A
        lambda: half(Xd, Zd, rp, cl, Ad[:50], dg, True, 1e-3, 0.01, order),                      # A per user
        lambda: half(Xd, Zd, rp, cl, Ad, dg.long(), True, 1e-3, 0.01, order),                   # int64 deg
        lambda: half(Xd, Zd, rp, cl, Ad, torch.cat([dg, dg]), True, 1e-3, 0.01, order),          # deg length
        lambda: half(Xd, Zd, rp, cl, Ad, dg - 3001, True, 1e-3, 0.01, order),                    # negative deg
        lambda: half(Zd, Xd, irp, icl, Ad, dg, False, 1e-3, 0.01, iorder, asum_out=Ad),          # asum_out is A
        lambda: half(Zd, Xd, irp, icl, Ad, dg, False, 1e-3, 0.01, iorder, asum_out=out.float()),  # float32 asum_out
        lambda: half(Xd, Zd, rp, cl, Ad, dg, True, 1e-3, 0.01, order, asum_out=out[:50]),       # sums need item rows
        lambda: half(Xd, Zd, rp[:-1], cl, Ad, dg, True, 1e-3, 0.01, order),                      # rowptr length
        lambda: half(Xd, Zd, rp, cl[:-1], Ad, dg, True, 1e-3, 0.01, order),                      # rowptr end
        lambda: half(Xd, Zd, rp, cl + 60, Ad, dg, True, 1e-3, 0.01, order),                      # column out of range
        lambda: half(Xd, Zd, rp, cl, Ad, dg, True, 1e-3, 0.01, order + 1),                       # row out of range
        lambda: half(Xd, Zd, rp, cl.long(), Ad, dg, True, 1e-3, 0.01, order),                    # int64 columns
        lambda: half(Xd.cpu(), Zd.cpu(), rp.cpu(), cl.cpu(), Ad.cpu(), dg.cpu(), True, 1e-3, 0.01, order.cpu()),
    ]
    for k, call in enumerate(bad):
        with pytest.raises(E.QRecError):
            call()
            pytest.fail('bad argument set %d was accepted' % k)
    assert np.array_equal(Xd.cpu().numpy(), theta) and np.array_equal(Zd.cpu().numpy(), beta)


def _golden_model(conf_extra, tmp_path, monkeypatch):
    from qrec_b200.model.ranking.SERec import SERec
    from qrec_b200.util.config import ModelConf
    g = np.load(GOLD)
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + conf_extra)
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    return g, SERec(conf, train, test, relation(g))


def test_dropin_reproduces_reference_run(torch, tmp_path, monkeypatch, capsys):
    """theta, beta and A after three epochs within the CPU oracle's bounds, the first epoch's mu print byte for byte,
    and the final measure lines."""
    g, model = _golden_model('', tmp_path, monkeypatch)
    measure = model.execute()
    text = capsys.readouterr().out
    with capsys.disabled():
        print('\ndrop-in measure', [m.strip() for m in measure], 'golden', g['measure'].tolist())
    assert 'epoch #0\n' + str(g['mu_str'][0]) + '\n\tUpdating exposure prior...\n' in text
    assert np.array_equal(model.deg, g['deg'])
    with capsys.disabled():
        _assert_golden(model.theta, model.beta, model.A, g, len(g['asum_epoch']) - 1)
    assert_measure(measure, g)


def test_gpu_eval_gives_the_host_top_n(torch, tmp_path, monkeypatch):
    """The device's top-10 lists are the host's up to the order of near-ties: at every rank the two items' host
    scores agree to a few float32 steps.  (Items rated by the same few users get nearly equal beta rows, so ties are
    common here; the two sides sum the float32 dot in different orders and break ties differently.)"""
    g, model = _golden_model('engine=-eval gpu\n', tmp_path, monkeypatch)
    measure = model.execute()
    _, N = model._top_n_setting()
    batched = model._recommend_all_on_device(N)
    assert batched is not None and len(batched) > 0
    same, worst = 0, 0.0
    for u, rec in batched.items():
        host = [n for n, _ in model._recommend(u, N)]
        dev = [n for n, _ in rec]
        if dev == host:
            same += 1
            continue
        s = np.asarray(model.predictForRanking(u), dtype=np.float64)
        ids = model.data.item
        gap = max(abs(s[ids[a]] - s[ids[b]]) for a, b in zip(dev, host)) / np.abs(s).max()
        worst = max(worst, gap)
    print('-eval gpu: %d of %d top-%d lists equal the host ones; the others swap near-ties (largest score gap %.2g '
          'of the largest score)' % (same, len(batched), N, worst))
    assert worst <= 5e-7
    assert_measure(measure, g)
