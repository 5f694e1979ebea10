"""Parity tests for K9 (the rating-prediction MF family, SURVEY.md §8 f-4): the CUDA path through the C
ABI against the pinned oracle and the golden runs of the reference's BasicMF / PMF / SVD.  Needs a GPU."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
REG = dict(reg_u=0.01, reg_i=0.02, reg_b=0.03)
NAMES = ['BasicMF', 'PMF', 'SVD']


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _load(name):
    g = np.load(os.path.join(GOLD, 'mf_%s_filmtrust.npz' % name.lower()))
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    u0 = np.array([users[x] for x in g['train_users'].tolist()], np.int32)
    i0 = np.array([items[x] for x in g['train_items'].tolist()], np.int32)
    return g, u0, i0


def _dev(torch, a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _ordered(torch, E, kind, P, Q, u, i, r, lr, Bu, Bi, gm, n_warps=0):
    wu, wi = E.mf_order_prepare(u, i, P.shape[0], Q.shape[0])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.mf_sgd_ordered(kind, P, Q, _dev(torch, u), _dev(torch, i), _dev(torch, r, P.dtype), _dev(torch, wu),
                     _dev(torch, wi), lr, REG['reg_u'], REG['reg_i'], loss, Bu, Bi, REG['reg_b'], gm, n_warps=n_warps)
    torch.cuda.synchronize()
    return float(loss.item())


@pytest.mark.parametrize('name', NAMES)
def test_ordered_f64_matches_reference_three_epochs(torch, E, name):
    """float64 parity mode == the reference's loop over all three golden epochs (visiting order, learning
    rate and loss assembly replayed on the host as the drop-in does)."""
    from oracle import bpr_oracle as O
    from oracle import mf_oracle as M
    g, u0, i0 = _load(name)
    kind = M.KINDS[name]
    P, Q = _dev(torch, g['P0']), _dev(torch, g['Q0'])
    Bu = _dev(torch, g['Bu0']) if kind == 2 else None
    Bi = _dev(torch, g['Bi0']) if kind == 2 else None
    gm = float(g['global_mean'])
    lr, last = float(g['lrate'][0][0]), 0.0
    for e in range(3):
        o = g['order_epoch'][e]
        sq = _ordered(torch, E, kind, P, Q, u0[o], i0[o], g['train_rating'][o], lr, Bu, Bi, gm)
        loss = M.epoch_loss(kind, sq, P.cpu().numpy(), Q.cpu().numpy(), REG['reg_u'], REG['reg_i'],
                            None if Bu is None else Bu.cpu().numpy(), None if Bi is None else Bi.cpu().numpy(),
                            REG['reg_b'])
        assert abs(loss - g['loss'][e]) <= 1e-9 * g['loss'][e]
        if not abs(last - loss) < 1e-3:
            lr = O.update_learning_rate(lr, 1.0, e + 1, last, loss)
        last = loss
    # the warp-shuffle dot groups the sum differently from numpy's ddot: last-bit noise over 100 K steps
    np.testing.assert_allclose(P.cpu().numpy(), g['P_last'], rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(Q.cpu().numpy(), g['Q_last'], rtol=1e-8, atol=1e-11)
    if kind == 2:
        np.testing.assert_allclose(Bu.cpu().numpy(), g['Bu_last'], rtol=1e-8, atol=1e-11)
        np.testing.assert_allclose(Bi.cpu().numpy(), g['Bi_last'], rtol=1e-8, atol=1e-11)


@pytest.mark.parametrize('name', NAMES)
@pytest.mark.parametrize('n_warps', [0, 16])
def test_ordered_f32_matches_sequential_f32_oracle(torch, E, name, n_warps):
    from oracle import c_oracle
    from oracle import mf_oracle as M
    g, u0, i0 = _load(name)
    kind = M.KINDS[name]
    n = 8000
    f32 = np.float32
    P0, Q0 = g['P0'].astype(f32), g['Q0'].astype(f32)
    Bu0 = g['Bu0'].astype(f32) if kind == 2 else None
    Bi0 = g['Bi0'].astype(f32) if kind == 2 else None
    gm = float(g['global_mean'])
    Pr, Qr = P0.copy(), Q0.copy()
    Bur, Bir = (Bu0.copy(), Bi0.copy()) if kind == 2 else (None, None)
    ref = c_oracle.mf_sgd_sequential(kind, Pr, Qr, u0[:n], i0[:n], g['train_rating'][:n], 0.02, REG['reg_u'],
                                     REG['reg_i'], Bur, Bir, REG['reg_b'], gm)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    Bu = _dev(torch, Bu0) if kind == 2 else None
    Bi = _dev(torch, Bi0) if kind == 2 else None
    got = _ordered(torch, E, kind, P, Q, u0[:n], i0[:n], g['train_rating'][:n], 0.02, Bu, Bi, gm, n_warps=n_warps)
    np.testing.assert_allclose(P.cpu().numpy(), Pr, rtol=2e-4, atol=2e-6)
    np.testing.assert_allclose(Q.cpu().numpy(), Qr, rtol=2e-4, atol=2e-6)
    if kind == 2:
        np.testing.assert_allclose(Bu.cpu().numpy(), Bur, rtol=2e-4, atol=2e-6)
    assert abs(got - ref) <= 1e-4 * ref


@pytest.mark.parametrize('kind', [0, 1, 2])
@pytest.mark.parametrize('d', [4, 12, 20, 64, 128])
def test_batch_kernel_equals_jacobi_step(torch, E, kind, d):
    """Throughput kernel.  (a) no row repeats inside the launch: Jacobi == sequential == the kernel, to fp32
    rounding.  (b) repeated rows: entries that are in flight together read the pre-launch rows (Jacobi), entries a
    lane group handles later in the launch already see the earlier deltas (sequential), so the result must lie in
    the band the two readings span (both differ from each other at second order in lr)."""
    from oracle import mf_oracle as M
    from oracle import c_oracle
    rng = np.random.default_rng(d * 3 + kind)
    nu, ni = 300, 200
    P0 = (rng.random((nu, d)) / 3).astype(np.float32); Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    Bu0 = (rng.random(nu) / 5).astype(np.float32); Bi0 = (rng.random(ni) / 5).astype(np.float32)
    for repeated in (False, True):
        n = 257 if repeated else 190
        if repeated:
            u = rng.integers(0, nu, n).astype(np.int32); i = rng.integers(0, ni, n).astype(np.int32)
        else:
            u = rng.permutation(nu)[:n].astype(np.int32); i = rng.permutation(ni)[:n].astype(np.int32)
        r = (rng.integers(1, 9, n) / 2.0).astype(np.float32)
        dP, dQ, dBu, dBi, ref = M.mf_sgd_jacobi(kind, P0, Q0, u, i, r, 0.01, 0.01, 0.02, Bu0, Bi0, 0.03, 3.0)
        Ps, Qs, Bus, Bis = P0.copy(), Q0.copy(), Bu0.copy(), Bi0.copy()
        ref_seq = c_oracle.mf_sgd_sequential(kind, Ps, Qs, u, i, r, 0.01, 0.01, 0.02, Bus if kind == 2 else None,
                                             Bis if kind == 2 else None, 0.03, 3.0)
        P, Q, Bu, Bi = (_dev(torch, a) for a in (P0, Q0, Bu0, Bi0))
        loss = torch.zeros(1, dtype=torch.float64, device='cuda')
        E.mf_sgd_batch(kind, P, Q, _dev(torch, u), _dev(torch, i), _dev(torch, r), 0.01, 0.01, 0.02, loss,
                       Bu if kind == 2 else None, Bi if kind == 2 else None, 0.03, 3.0)
        torch.cuda.synchronize()
        pairs = [(P.cpu().numpy(), P0 + dP, Ps), (Q.cpu().numpy(), Q0 + dQ, Qs)]
        if kind == 2:
            pairs += [(Bu.cpu().numpy(), Bu0 + dBu, Bus), (Bi.cpu().numpy(), Bi0 + dBi, Bis)]
        else:
            assert np.array_equal(Bu.cpu().numpy(), Bu0)
        for got, jac, seq in pairs:
            if not repeated:
                np.testing.assert_allclose(got, jac, rtol=2e-5, atol=2e-6)
                np.testing.assert_allclose(got, seq, rtol=2e-5, atol=2e-6)
            else:
                band = float(np.abs(jac - seq).max())
                assert band > 0
                # not strictly inside the band: an entry may see some but not all earlier deltas of a shared row
                assert float(np.abs(got - jac).max()) <= 1.5 * band + 5e-6
                assert float(np.abs(got - seq).max()) <= 1.5 * band + 5e-6
        lo, hi = min(ref, ref_seq), max(ref, ref_seq)
        assert lo * (1 - 1e-5) <= float(loss.item()) <= hi * (1 + 1e-5)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_predict_pairs(torch, E, dtype):
    rng = np.random.default_rng(1)
    P = rng.random((50, 20)).astype(dtype); Q = rng.random((70, 20)).astype(dtype)
    Bu = rng.random(50).astype(dtype); Bi = rng.random(70).astype(dtype)
    u = rng.integers(0, 50, 1000).astype(np.int32); i = rng.integers(0, 70, 1000).astype(np.int32)
    got = E.mf_predict_pairs(_dev(torch, P), _dev(torch, Q), _dev(torch, u), _dev(torch, i)).cpu().numpy()
    tol = 1e-5 if dtype == 'float32' else 1e-12
    np.testing.assert_allclose(got, (P[u] * Q[i]).sum(1), rtol=tol)
    got = E.mf_predict_pairs(_dev(torch, P), _dev(torch, Q), _dev(torch, u), _dev(torch, i), _dev(torch, Bu),
                             _dev(torch, Bi), 2.5).cpu().numpy()
    np.testing.assert_allclose(got, (P[u] * Q[i]).sum(1) + 2.5 + Bi[i] + Bu[u], rtol=tol)


def test_edges(torch, E):
    P = torch.zeros(4, 8, device='cuda'); Q = torch.zeros(5, 8, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    empty_i = torch.zeros(0, dtype=torch.int32, device='cuda'); empty_f = torch.zeros(0, device='cuda')
    E.mf_sgd_batch(1, P, Q, empty_i, empty_i, empty_f, 0.1, 0.0, 0.0, loss)           # n = 0: no-op
    E.mf_sgd_ordered(1, P, Q, empty_i, empty_i, empty_f, empty_i, empty_i, 0.1, 0.0, 0.0, loss)
    assert float(loss.item()) == 0.0 and float(P.abs().sum().item()) == 0.0
    one = torch.zeros(1, dtype=torch.int32, device='cuda'); rf = torch.ones(1, device='cuda')
    with pytest.raises(E.QRecError):
        E.mf_sgd_batch(3, P, Q, one, one, rf, 0.1, 0.0, 0.0, loss)                    # unknown kind
    with pytest.raises(E.QRecError):
        E.mf_sgd_batch(2, P, Q, one, one, rf, 0.1, 0.0, 0.0, loss)                    # SVD without biases
    P10 = torch.zeros(4, 10, device='cuda'); Q10 = torch.zeros(5, 10, device='cuda')
    with pytest.raises(E.QRecError):
        E.mf_sgd_batch(1, P10, Q10, one, one, rf, 0.1, 0.0, 0.0, loss)                # d % 4 != 0
    # a single entry: e = 1 - 0, rows stay zero under kind 1 (e*q = 0), loss = 1
    E.mf_sgd_batch(1, P, Q, one, one, rf, 0.1, 0.0, 0.0, loss)
    torch.cuda.synchronize()
    assert float(loss.item()) == 1.0


@pytest.mark.parametrize('window', [1, 64, 100000])
def test_batch_kernel_window_only_changes_the_grid(torch, E, window):
    """max_inflight sizes the grid, not the result: on a launch without repeated rows every window
    gives the Jacobi (= sequential) update."""
    from oracle import mf_oracle as M
    rng = np.random.default_rng(window)
    nu, ni, n, d = 3000, 2500, 2000, 32
    P0 = (rng.random((nu, d)) / 3).astype(np.float32); Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    u = rng.permutation(nu)[:n].astype(np.int32); i = rng.permutation(ni)[:n].astype(np.int32)
    r = (rng.integers(1, 9, n) / 2.0).astype(np.float32)
    dP, dQ, _, _, ref = M.mf_sgd_jacobi(1, P0, Q0, u, i, r, 0.01, 0.01, 0.02)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.mf_sgd_batch(1, P, Q, _dev(torch, u), _dev(torch, i), _dev(torch, r), 0.01, 0.01, 0.02, loss, max_inflight=window)
    torch.cuda.synchronize()
    np.testing.assert_allclose(P.cpu().numpy(), P0 + dP, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(Q.cpu().numpy(), Q0 + dQ, rtol=2e-5, atol=2e-6)
    assert abs(float(loss.item()) - ref) <= 1e-5 * ref


@pytest.mark.parametrize('name', NAMES)
def test_dropin_parity_mode_reproduces_reference_run(torch, name, tmp_path, monkeypatch):
    """The drop-in class, default engine mode (parity, float64), from the same seeds as the golden run:
    tables, epoch losses, learning rates and the MAE / RMSE lines of the reference."""
    import importlib
    import random
    from qrec_b200.util.config import ModelConf
    g = np.load(os.path.join(GOLD, 'mf_%s_filmtrust.npz' % name.lower()))
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']))
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    cls = getattr(importlib.import_module('qrec_b200.model.rating.' + name), name)
    model = cls(conf, train, test)
    losses = []
    orig = cls.isConverged
    monkeypatch.setattr(cls, 'isConverged', lambda self, ep: (losses.append(self.loss), orig(self, ep))[1])
    measure = model.execute()
    np.testing.assert_allclose(model.P, g['P_last'], rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(model.Q, g['Q_last'], rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(losses, g['loss'], rtol=1e-9)
    for got, ref in zip(measure, g['measure'].tolist()):
        assert got.split(':')[0] == ref.split(':')[0]
        assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-6


@pytest.mark.parametrize('name', ['PMF', 'SVD'])
def test_dropin_fast_mode_lands_near_reference_error(torch, name, tmp_path, monkeypatch):
    import importlib
    import random
    from qrec_b200.util.config import ModelConf
    g = np.load(os.path.join(GOLD, 'mf_%s_filmtrust.npz' % name.lower()))
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + 'engine=-mode fast\n')
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    cls = getattr(importlib.import_module('qrec_b200.model.rating.' + name), name)
    measure = cls(conf, train, test).execute()
    rmse = float(measure[1].strip().split(':')[1])
    assert abs(rmse - float(str(g['measure'][1]).split(':')[1])) < 0.05
