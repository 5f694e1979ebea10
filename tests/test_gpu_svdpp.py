"""K11 (SVD++) on the GPU: qrec_svdpp_sgd_ordered_* against the golden run of the reference's SVD++
(tests/golden/svdpp_filmtrust.npz) and the numpy oracle (oracle/svdpp_oracle.py), qrec_svdpp_epoch_usermajor_f32
against the oracle's per-user closed form, and the drop-in.  Needs a GPU."""
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import svdpp_oracle as S          # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'svdpp_filmtrust.npz')
REG = dict(reg_u=0.01, reg_i=0.01, reg_b=0.1, reg_y=0.01)        # SVD++.conf
REGS = (REG['reg_u'], REG['reg_i'], REG['reg_b'], REG['reg_y'])
TABLES = ('P', 'Q', 'Y', 'Bu', 'Bi')


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def ids(g):
    return S.golden_ids(g)


def _dev(torch, a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t.to(dtype) if dtype is not None else t


def _ordered(torch, E, tabs, u, i, r, csr, lr, gm):
    dt = tabs[0].dtype
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.svdpp_sgd_ordered(*tabs, _dev(torch, u.astype(np.int32)), _dev(torch, i.astype(np.int32)), _dev(torch, r, dt),
                        _dev(torch, csr[0]), _dev(torch, csr[1]), lr, *REGS, gm, loss)
    return float(loss.item())


def test_ordered_f64_reproduces_golden_epochs(torch, E, g, ids):
    """Three epochs in the recorded visiting orders: all five tables after every epoch (rtol 1e-8) and the loss
    (1e-9).  The only difference from the reference is how the two dot products' partial sums are grouped."""
    u0, i0, csr, _, _ = ids
    tabs = [_dev(torch, t) for t in S.initial_tables(g)]
    gm = float(g['global_mean'])
    k = int(g['row_stride'])
    for e in range(len(g['loss'])):
        o = g['order_epoch'][e].astype(np.int64)
        sq = _ordered(torch, E, tabs, u0[o], i0[o], g['train_rating'][o], csr, float(g['lrate'][e][0]), gm)
        host = [t.cpu().numpy() for t in tabs]
        loss = S.epoch_loss(sq, *host, *REGS)
        assert abs(loss - g['loss'][e]) <= 1e-9 * g['loss'][e]
        for name, t in zip(TABLES, host):
            ref = g[name + '_rows_epoch'][e]
            np.testing.assert_allclose(t[::k], ref, rtol=1e-8, atol=1e-10 * float(np.abs(ref).max()))
            if e == len(g['loss']) - 1:
                ref = g[name + '_last']
                np.testing.assert_allclose(t, ref, rtol=1e-8, atol=1e-10 * float(np.abs(ref).max()))


def test_ordered_f32_tracks_the_f32_oracle(torch, E, g, ids):
    u0, i0, csr, _, _ = ids
    n = 8000
    init = [t.astype(np.float32) for t in S.initial_tables(g)]
    tabs = [_dev(torch, t) for t in init]
    gm = float(g['global_mean'])
    r = g['train_rating'][:n]
    sq = _ordered(torch, E, tabs, u0[:n], i0[:n], r, csr, 0.02, gm)
    ref = [t.copy() for t in init]
    rsq = S.svdpp_sgd_sequential(*ref, u0[:n], i0[:n], r, csr[0], csr[1], 0.02, *REGS, gm)
    for t, x in zip(tabs, ref):
        np.testing.assert_allclose(t.cpu().numpy(), x, rtol=2e-4, atol=2e-6)
    assert abs(sq - rsq) <= 1e-4 * rsq


def _problem(seed, nu, ni, d, deg_max, disjoint=False):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, deg_max + 1, nu)
    rowptr = np.zeros(nu + 1, dtype=np.int64)
    np.cumsum(lengths, out=rowptr[1:])
    if disjoint:
        assert rowptr[-1] <= ni
        cols = rng.permutation(ni)[:rowptr[-1]].astype(np.int32)
    else:
        cols = np.concatenate([rng.choice(ni, k, replace=False) for k in lengths]).astype(np.int32)
    vals = rng.integers(1, 9, len(cols)) / 2.0
    tabs = [rng.random((nu, d)) / 3, rng.random((ni, d)) / 3, rng.random((ni, d)), rng.random(nu), rng.random(ni)]
    return tabs, (rowptr, cols, vals)


@pytest.mark.parametrize('d', [1, 37, 256])
def test_ordered_f64_any_width(torch, E, d):
    """d from 1 to 256, users with one item and long rows that span several staged chunks."""
    tabs, csr = _problem(d, 40, 3000, d, 300 if d == 256 else 60)
    u, i, r = S.user_entries(*csr, np.arange(40, dtype=np.int32))
    perm = np.random.default_rng(d).permutation(len(u))
    u, i, r = u[perm], i[perm], r[perm]
    dev_tabs = [_dev(torch, t) for t in tabs]
    sq = _ordered(torch, E, dev_tabs, u, i, r, csr, 0.01, 2.5)
    rsq = S.svdpp_sgd_sequential(*tabs, u, i, r, csr[0], csr[1], 0.01, *REGS, 2.5)
    for t, x in zip(dev_tabs, tabs):
        np.testing.assert_allclose(t.cpu().numpy(), x, rtol=1e-8, atol=1e-11)
    assert abs(sq - rsq) <= 1e-9 * rsq


def test_ordered_rejects_wide_tables_and_skips_empty_epochs(torch, E):
    tabs, csr = _problem(3, 5, 50, 257, 4)
    u, i, r = S.user_entries(*csr, np.arange(5, dtype=np.int32))
    with pytest.raises(E.QRecError):
        _ordered(torch, E, [_dev(torch, t) for t in tabs], u, i, r, csr, 0.01, 2.5)
    tabs, csr = _problem(3, 5, 50, 8, 4)
    before = E.launch_count()
    assert _ordered(torch, E, [_dev(torch, t) for t in tabs], u[:0], i[:0], r[:0], csr, 0.01, 2.5) == 0.0
    assert E.launch_count() == before


def _fast(torch, E, tabs, csr, order, lr, gm, in_flight, dpad=None):
    d = tabs[0].shape[1]
    dpad = dpad or d

    def up(a):
        if a.ndim == 1:
            return _dev(torch, a.astype(np.float32))
        t = torch.zeros(a.shape[0], dpad, dtype=torch.float32, device='cuda')
        t[:, :d] = _dev(torch, a.astype(np.float32))
        return t
    dev_tabs = [up(t) for t in tabs]
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.svdpp_epoch_usermajor(*dev_tabs, _dev(torch, csr[0]), _dev(torch, csr[1]), _dev(torch, csr[2], torch.float32),
                            _dev(torch, order), lr, *REGS, gm, loss, max_users_in_flight=in_flight)
    return [t.cpu().numpy() for t in dev_tabs], float(loss.item())


def _oracle_fast(tabs, csr, order, lr, gm):
    ref = [t.astype(np.float32).astype(np.float64) for t in tabs]
    loss = S.svdpp_usermajor(*ref, *csr, order, lr, *REGS, gm)
    return ref, loss


def test_fast_one_user_in_flight_is_the_closed_form(torch, E, g, ids):
    """FilmTrust, d = 10 padded to 12, users longest first, one user at a time: the float64 closed form to the K9
    fp32 tolerance; the padding columns stay zero."""
    _, _, csr, _, _ = ids
    order = E.als_row_order(csr[0])
    init = S.initial_tables(g)
    gm = float(g['global_mean'])
    got, loss = _fast(torch, E, init, csr, order, 0.02, gm, 1, dpad=12)
    ref, rloss = _oracle_fast(init, csr, order, 0.02, gm)
    for t, x in zip(got, ref):
        if t.ndim == 2:
            assert not t[:, 10:].any()
            t = t[:, :10]
        np.testing.assert_allclose(t, x, rtol=2e-4, atol=2e-6)
    assert abs(loss - rloss) <= 1e-4 * rloss


@pytest.mark.parametrize('d', [4, 64, 128])
def test_fast_full_concurrency_disjoint_users_is_the_closed_form(torch, E, d):
    """Users that share no item do not interact, so filling the GPU gives the one-at-a-time result."""
    tabs, csr = _problem(d, 3000, 3000 * 12, d, 12, disjoint=True)
    order = E.als_row_order(csr[0])
    got, loss = _fast(torch, E, tabs, csr, order, 0.02, 3.0, 0)
    ref, rloss = _oracle_fast(tabs, csr, order, 0.02, 3.0)
    for t, x in zip(got, ref):
        np.testing.assert_allclose(t, x, rtol=2e-4, atol=2e-6)
    assert abs(loss - rloss) <= 1e-4 * rloss


def test_fast_rejects_wide_or_unpadded_tables_and_skips_empty_epochs(torch, E):
    for d in (132, 10):
        tabs, csr = _problem(5, 10, 200, d, 5)
        with pytest.raises(E.QRecError):
            _fast(torch, E, tabs, csr, np.arange(10, dtype=np.int32), 0.02, 3.0, 0)
    tabs, csr = _problem(5, 10, 200, 8, 5)
    before = E.launch_count()
    got, loss = _fast(torch, E, tabs, csr, np.arange(0, dtype=np.int32), 0.02, 3.0, 0)
    assert E.launch_count() == before and loss == 0.0
    np.testing.assert_array_equal(got[0], tabs[0].astype(np.float32))


def _golden_model(g, conf_extra, tmp_path, monkeypatch):
    from qrec_b200.model.rating.SVDPlusPlus import SVDPlusPlus
    from qrec_b200.util.config import ModelConf
    monkeypatch.chdir(tmp_path)
    conf = ModelConf.from_string(str(g['conf']) + conf_extra)
    train = [[u, i, r] for u, i, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())]
    test = [[u, i, r] for u, i, r in zip(g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())]
    random.seed(int(g['seed'])); np.random.seed(int(g['seed']))
    return SVDPlusPlus(conf, train, test)


def _lines_close(got, ref):
    assert [m.split(':')[0] for m in got] == [m.split(':')[0] for m in ref]
    for a, b in zip(got, ref):
        assert abs(float(a.split(':')[1]) - float(b.split(':')[1])) < 1e-6


def test_dropin_parity_reproduces_reference_run(torch, g, tmp_path, monkeypatch):
    """Default engine (float64, ordered kernel) from the golden seeds: the five tables, the epoch losses, learning
    rates, MT19937 states and every MAE / RMSE line."""
    model = _golden_model(g, '', tmp_path, monkeypatch)
    cls = type(model)
    seen = []
    orig = cls.isConverged

    def spy(self, epoch):
        lr0 = self.lRate
        r = orig(self, epoch)
        seen.append((self.loss, lr0, self.lRate, np.array(random.getstate()[1], dtype=np.uint32),
                     [m.strip() for m in self.measure]))
        return r
    monkeypatch.setattr(cls, 'isConverged', spy)
    measure = model.execute()
    for name in TABLES:
        ref = g[name + '_last']
        np.testing.assert_allclose(getattr(model, name), ref, rtol=1e-8, atol=1e-10 * float(np.abs(ref).max()))
    assert len(seen) == len(g['loss'])
    for e, (loss, lr0, lr1, st, lines) in enumerate(seen):
        assert abs(loss - g['loss'][e]) <= 1e-9 * g['loss'][e]
        assert (lr0, lr1) == tuple(g['lrate'][e])
        assert np.array_equal(st, g['mt_state_after_epoch'][e])
        _lines_close(lines, g['epoch_measure'][e].tolist())
    _lines_close([m.strip() for m in measure], g['measure'].tolist())


def test_dropin_fast_mode_lands_near_reference(torch, g, tmp_path, monkeypatch):
    model = _golden_model(g, 'engine=-mode fast\n', tmp_path, monkeypatch)
    measure = model.execute()
    assert model.Y.shape == g['Y_last'].shape and np.isfinite(model.Y).all()
    rmse = float(measure[1].strip().split(':')[1])
    ref = float(str(g['measure'][1]).split(':')[1])
    assert abs(rmse - ref) < 0.05


def test_module_entry_point_runs_the_svdpp_conf(torch, g, tmp_path, monkeypatch, capsys):
    """`python -m qrec_b200 SVD++.conf`: the shipped configuration (60 epochs, parity engine) from files on disk."""
    monkeypatch.chdir(tmp_path)
    os.makedirs('dataset/FilmTrust')
    for name, pre in (('trainset.txt', 'train'), ('testset.txt', 'test')):
        with open('dataset/FilmTrust/' + name, 'w') as f:
            for u, i, r in zip(g[pre + '_users'].tolist(), g[pre + '_items'].tolist(), g[pre + '_rating'].tolist()):
                f.write('%s %s %s\n' % (u, i, r))
    with open('SVD++.conf', 'w') as f:
        f.write(str(g['conf']).replace('num.max.epoch=3', 'num.max.epoch=60'))
    from qrec_b200.__main__ import main
    measure = main(['SVD++.conf', '--seed', str(int(g['seed']))])
    out = capsys.readouterr().out
    assert 'Running time:' in out and 'epoch 60:' in out
    mae, rmse = (float(m.strip().split(':')[1]) for m in measure[:2])
    assert 0.5 < mae < 0.8 and 0.6 < rmse < 1.0
