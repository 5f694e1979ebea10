"""K10 (WRMF, implicit-feedback ALS) on the GPU: qrec_als_gram_* and qrec_als_solve_rows_* against numpy and the
oracle (oracle/wrmf_oracle.py), and the drop-in against the golden run of the reference's WRMF
(tests/golden/wrmf_filmtrust.npz).  Needs a GPU."""
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import wrmf_oracle as W          # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'wrmf_filmtrust.npz')
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


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('d', DS)
@pytest.mark.parametrize('n', [0, 1, 1000, 300001])
def test_gram_matches_numpy_and_is_bitwise_stable(torch, E, dtype, d, n):
    rng = np.random.default_rng(n * 131 + d)
    Z = (rng.random((n, d)) / 3).astype(dtype)
    Zt = _dev(torch, Z)
    G1 = E.als_gram(Zt).cpu().numpy()
    G2 = E.als_gram(Zt).cpu().numpy()
    Z64 = Z.astype(np.float64)
    np.testing.assert_allclose(G1, Z64.T @ Z64, rtol=1e-12, atol=0)
    assert np.array_equal(G1, G2) and np.array_equal(G1, G1.T)


def _problem(d, seed, n_z=60000, long_row=50000):
    """40 rows to solve against n_z rows of Z: lengths 0, 1, 5..60 and one of `long_row` entries."""
    rng = np.random.default_rng(seed)
    Z = rng.random((n_z, d)) / 3
    lengths = np.concatenate([[0, 1], rng.integers(5, 61, 37), [long_row]])
    rowptr = np.zeros(len(lengths) + 1, dtype=np.int64)
    np.cumsum(lengths, out=rowptr[1:])
    cols = np.concatenate([rng.choice(n_z, k, replace=False) for k in lengths]).astype(np.int32)
    vals = rng.integers(1, 6, len(cols)).astype(np.float64)
    X = rng.random((len(lengths), d)) / 3
    return X, Z, rowptr, cols, vals


def _solve(torch, E, X, Z, rowptr, cols, vals, lam, dtype, loss=True):
    Xt, Zt = _dev(torch, X.astype(dtype)), _dev(torch, Z.astype(dtype))
    G = E.als_gram(Zt)
    acc = torch.zeros(1, dtype=torch.float64, device='cuda') if loss else None
    order = _dev(torch, E.als_row_order(rowptr))
    E.als_solve_rows(Xt, Zt, G, _dev(torch, rowptr), _dev(torch, cols), _dev(torch, vals.astype(dtype)), lam, W.ALPHA,
                     order, loss=acc)
    return Xt.cpu().numpy(), (float(acc.item()) if loss else None)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('d', DS)
def test_solve_rows_matches_oracle(torch, E, dtype, d):
    X, Z, rowptr, cols, vals = _problem(d, seed=d)
    Xq, Zq = X.astype(dtype).astype(np.float64), Z.astype(dtype).astype(np.float64)
    ref = Xq.copy()
    ref_loss = W.solve_side(ref, Zq, rowptr, cols, vals, 1.0, with_loss=True)
    got, loss = _solve(torch, E, X, Z, rowptr, cols, vals, 1.0, dtype)
    got2, _ = _solve(torch, E, X, Z, rowptr, cols, vals, 1.0, dtype)
    assert np.array_equal(got, got2)
    assert np.array_equal(got[0], np.zeros(d))                       # no entries: (G + lambda I) x = 0
    scale = float(np.abs(ref).max())
    if dtype == 'float64':
        np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12 * scale)
    else:
        np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-6 * scale)
    assert abs(loss - ref_loss) <= 1e-12 * ref_loss


def test_solve_rows_rejects_wide_rows_and_reports_indefinite_systems(torch, E):
    X, Z, rowptr, cols, vals = _problem(129, seed=5, n_z=200, long_row=150)
    with pytest.raises(E.QRecError):
        _solve(torch, E, X, Z, rowptr, cols, vals, 1.0, 'float64')
    X, Z, rowptr, cols, vals = _problem(20, seed=6, n_z=2000, long_row=1500)
    Xt, Zt = _dev(torch, X), _dev(torch, Z)
    G = E.als_gram(Zt)
    order = _dev(torch, E.als_row_order(rowptr))
    args = (Xt, Zt, G, _dev(torch, rowptr), _dev(torch, cols), _dev(torch, vals))
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    # lambda far below -(largest eigenvalue of A without it): every row's A is negative definite
    E.als_solve_rows(*args, -1e9, W.ALPHA, order, n_failed=n_failed)
    assert int(n_failed.item()) == X.shape[0]
    assert np.array_equal(Xt.cpu().numpy(), X)
    with pytest.raises(E.QRecError):
        E.als_solve_rows(*args, -1e9, W.ALPHA, order)
    assert np.array_equal(Xt.cpu().numpy(), X)


def _golden_model(conf_extra, tmp_path, monkeypatch):
    from qrec_b200.model.ranking.WRMF import WRMF
    from qrec_b200.util.config import ModelConf
    g = np.load(GOLD)
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + conf_extra)
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    return g, WRMF, WRMF(conf, train, test)


def test_dropin_reproduces_reference_run(torch, tmp_path, monkeypatch):
    """Default engine (float64 tables) from the golden seeds: tables after three epochs, epoch losses, learning
    rates and MT19937 state after every epoch, and the final measure lines."""
    g, cls, model = _golden_model('', tmp_path, monkeypatch)
    seen = []
    orig = cls.isConverged

    def spy(self, epoch):
        lr0 = self.lRate
        r = orig(self, epoch)
        seen.append((self.loss, lr0, self.lRate, np.array(random.getstate()[1], dtype=np.uint32)))
        return r
    monkeypatch.setattr(cls, 'isConverged', spy)
    measure = model.execute()
    for got, ref in ((model.X, g['X_last']), (model.Y, g['Y_last'])):
        np.testing.assert_allclose(got, ref, rtol=1e-8, atol=1e-10 * float(np.abs(ref).max()))
    assert len(seen) == len(g['loss'])
    for e, (loss, lr0, lr1, st) in enumerate(seen):
        assert abs(loss - g['loss'][e]) <= 1e-9 * g['loss'][e]
        assert (lr0, lr1) == tuple(g['lrate'][e])
        assert np.array_equal(st, g['mt_state_after_epoch'][e])
    for got, ref in zip(measure, g['measure'].tolist()):
        assert got.strip().split(':')[0] == ref.split(':')[0]
        if ':' in ref:
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-6


def test_dropin_fast_mode_with_gpu_eval_lands_near_reference(torch, tmp_path, monkeypatch):
    g, _, model = _golden_model('engine=-mode fast -eval gpu\n', tmp_path, monkeypatch)
    measure = model.execute()
    got = {m.split(':')[0]: float(m.split(':')[1]) for m in measure if ':' in m}
    ref = {m.split(':')[0]: float(m.split(':')[1]) for m in g['measure'].tolist() if ':' in m}
    for k in ('Precision', 'Recall'):
        assert abs(got[k] - ref[k]) < 0.01
