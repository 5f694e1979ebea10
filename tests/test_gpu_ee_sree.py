"""EE (K9 kind 5) and SREE (K9 kind 5 + the SREE pass of K17) on the GPU against the reference's golden runs and the
numpy oracle."""
import contextlib
import gzip
import io
import os
import random
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import ee_sree_oracle as EO             # noqa: E402
from oracle import socialmf_soreg_oracle as SM      # noqa: E402
from test_ee_sree_cpu import (GOLD, TAGS, case_files, cases, film, hyper, initial, load_run, model_of,  # noqa: E402
                              social_of, wrapper_cases)
from test_social_rating_cpu import conf_value, orders   # noqa: E402
from test_socialmf_soreg_cpu import _csr, _random_graph   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _dev(torch, a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


class SreePass(object):
    """SREE's user pass through the engine wrapper, on device tables of one dtype."""

    def __init__(self, torch, E, U, visit, fl, gl, dtype):
        self.t, self.E = torch, E
        fr, fc = _csr([ids for ids, _ in fl])
        fw = np.array([w for _, ws in fl for w in ws], np.float64)
        gr, gc = _csr([ids for ids, _ in gl])
        visit = np.asarray(visit, np.int32)
        pos, self.depth = E.social_order_prepare(visit, U, fr, fc, gr, gc)
        self.args = (_dev(torch, visit), _dev(torch, pos), _dev(torch, fr), _dev(torch, fc), _dev(torch, fw, dtype),
                     _dev(torch, gr), _dev(torch, gc))

    def __call__(self, P, lr, alpha, n_warps=0):
        loss = self.t.zeros(1, dtype=self.t.float64, device='cuda')
        self.E.sree_user_pass(P, *self.args, lr, alpha, loss, n_warps=n_warps)
        return float(loss.item())


def _rating_pass(torch, E, tables, u, i, r, lr, h, n_warps=0):
    P, Q, Bu, Bi = tables
    wu, wi = E.mf_order_prepare(u, i, P.shape[0], Q.shape[0])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.mf_sgd_ordered(E.EE_RATINGS, P, Q, _dev(torch, u), _dev(torch, i), _dev(torch, r, P.dtype), _dev(torch, wu),
                     _dev(torch, wi), lr, h['reg_u'], h['reg_i'], loss, Bu, Bi, h['reg_b'], h['global_mean'],
                     n_warps=n_warps)
    return float(loss.item())


def _replay_on_device(torch, E, g):
    """Every recorded epoch on the device (float64).  After each rating pass SREE's user pass also runs in the oracle
    on the same input rows, and the two must agree bit for bit.  Returns (tables after epoch 1, after the last epoch,
    losses)."""
    users, items, u0, i0 = load_run(g)
    h = hyper(g)
    tables = [_dev(torch, t) for t in initial(g)]
    sp = None
    if model_of(g) == 'SREE':
        visit, fl, gl, _ = social_of(g)
        sp = SreePass(torch, E, len(users), visit, fl, gl, torch.float64)
        alpha = conf_value(g, 'SREE', '-alpha')
    losses, first = [], None
    for e, o in enumerate(orders(g)):
        lr = float(g['lrate'][e][0])
        loss = _rating_pass(torch, E, tables, u0[o], i0[o], g['train_rating'][o], lr, h)
        host = [t.cpu().numpy() for t in tables]
        loss += float(EO.bias_penalty(host[2], host[3], h['reg_b']))
        if sp is not None:
            Ph = host[0].copy()
            social = sp(tables[0], lr, alpha)
            want = EO.sree_user_pass(Ph, visit, fl, lr, alpha)
            assert np.array_equal(tables[0].cpu().numpy(), Ph), 'user pass != oracle, epoch %d' % (e + 1)
            assert abs(social - float(want)) <= 1e-12 * max(1.0, abs(float(want)))
            loss += social
        losses.append(loss)
        if e == 0:
            first = [t.cpu().numpy().copy() for t in tables]
    return first, [t.cpu().numpy() for t in tables], losses


def _check_f64(torch, E, g):
    first, last, losses = _replay_on_device(torch, E, g)
    # K9's distance is a warp tree sum, not numpy's: tables and biases agree with the reference to rounding
    for t, k in zip(first, ('P', 'Q', 'Bu', 'Bi')):
        np.testing.assert_allclose(t.astype(np.float32), g[k + '_epoch1'], rtol=1e-6, atol=1e-7)
    for t, k in zip(last, ('P', 'Q', 'Bu', 'Bi')):
        np.testing.assert_allclose(t, g[k + '_last'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(losses, g['loss'], rtol=1e-12)


@pytest.mark.parametrize('name', ['EE', 'SREE'])
def test_f64_kernels_reproduce_the_reference_filmtrust_run(torch, E, name):
    _check_f64(torch, E, film(name))


@pytest.mark.parametrize('tag', TAGS)
def test_f64_kernels_reproduce_the_constructed_runs(torch, E, tag):
    _check_f64(torch, E, cases()[tag])


@pytest.mark.parametrize('name', ['EE', 'SREE'])
def test_f32_kernels_match_the_f32_oracle(torch, E, name):
    g = film(name)
    users, _, u0, i0 = load_run(g)
    h = hyper(g)
    host = initial(g, np.float32)
    tables = [_dev(torch, t.copy()) for t in host]
    o = orders(g)[1]
    u, i, r = u0[o], i0[o], g['train_rating'][o]
    lr = float(g['lrate'][0][0])
    _rating_pass(torch, E, tables, u, i, r, lr, h)
    if name == 'SREE':
        visit, fl, gl, _ = social_of(g)
        alpha = conf_value(g, 'SREE', '-alpha')
        SreePass(torch, E, len(users), visit, fl, gl, torch.float32)(tables[0], lr, alpha)
        EO.sree_epoch(*host, u, i, r, visit, fl, lr, h['reg_u'], h['reg_i'], h['reg_b'], h['global_mean'], alpha)
    else:
        EO.ee_epoch(*host, u, i, r, lr, h['reg_u'], h['reg_i'], h['reg_b'], h['global_mean'])
    for t, want in zip(tables, host):
        assert t.dtype == torch.float32
        np.testing.assert_allclose(t.cpu().numpy(), want, rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('d', [1, 40, 70, 100, 150, 190, 210, 256])
def test_result_does_not_depend_on_the_grid(torch, E, dtype, d):
    """One d per lane shape (E = 1..8, ragged widths included).  The rating pass over a stream with many repeated rows,
    and SREE's pass over a dense trust graph (up to 24 followees per user, a self-follow, zero weights) with a visiting
    order that skips some users: n_warps 1 (one CTA of 8 warps) and the full grid give the same bits; the user pass
    also gives the bits of the sequential oracle in the same precision."""
    U, I, n = 200, 150, 6000
    rs = np.random.RandomState(d)
    dt = getattr(torch, dtype)
    npdt = np.float64 if dtype == 'float64' else np.float32
    u = rs.randint(0, U, n).astype(np.int32)
    i = rs.randint(0, I, n).astype(np.int32)
    r = (0.5 * rs.randint(1, 9, n)).astype(np.float64)
    h = dict(reg_u=0.01, reg_i=0.02, reg_b=0.03, global_mean=2.5)
    init = [(rs.rand(U, d) / (3 * d)).astype(npdt), (rs.rand(I, d) / (3 * d)).astype(npdt),
            (rs.rand(U) / 10).astype(npdt), (rs.rand(I) / 10).astype(npdt)]
    out = []
    for n_warps in (1, 0):
        tables = [_dev(torch, t.copy()) for t in init]
        loss = _rating_pass(torch, E, tables, u, i, r, 0.005, h, n_warps=n_warps)
        out.append(([t.cpu().numpy() for t in tables], loss))
    for a, b in zip(out[0][0], out[1][0]):
        assert np.array_equal(a, b)
    assert abs(out[0][1] - out[1][1]) <= 1e-12 * abs(out[0][1])

    followees, followers = _random_graph(rs, U, 24)
    ws = {(a, b): float(np.round(rs.rand(), 2)) for a in range(U) for b in followees[a]}
    for b in followees[2]:
        ws[(2, b)] = 0.0
    fl = [(followees[a], [ws[(a, b)] for b in followees[a]]) for a in range(U)]
    gl = [(followers[b], [ws[(a, b)] for a in followers[b]]) for b in range(U)]
    visit = [int(x) for x in rs.permutation(U)[:180]]
    sp = SreePass(torch, E, U, visit, fl, gl, dt)
    P0 = (rs.rand(U, d) / 3).astype(npdt)
    res = []
    for n_warps in (1, 0):
        P = _dev(torch, P0.copy())
        loss = sp(P, 0.01, 0.5, n_warps=n_warps)
        res.append((P.cpu().numpy(), loss))
    assert np.array_equal(res[0][0], res[1][0])
    assert abs(res[0][1] - res[1][1]) <= 1e-12 * abs(res[0][1])
    Ph = P0.copy()
    want = EO.sree_user_pass(Ph, visit, fl, 0.01, 0.5)
    assert np.array_equal(res[0][0], Ph)
    assert abs(res[0][1] - float(want)) <= (1e-12 if dtype == 'float64' else 1e-5) * abs(float(want))
    assert sp.depth == SM.schedule(visit, U, followees, followers)[1]


def test_wrappers_raise_qrecerror_on_each_invalid_input(torch, E):
    """The valid call runs; every invalid input, shapes and contents alike, raises its own QRecError."""
    ok, bad = wrapper_cases(torch, 'cuda')
    E.sree_user_pass(**ok)
    torch.cuda.synchronize()
    assert float(ok['loss'].item()) > 0
    for k, (call, message, _) in enumerate(bad):
        with pytest.raises(E.QRecError, match=message):
            call()
            pytest.fail('case %d did not raise' % k)


# ------------------------------------------------------------------------------------------------ drop-ins
def _write_inputs(g, tmp_path, conf, case=False):
    if case:
        for name, lines in case_files().items():
            (tmp_path / name).write_text('\n'.join(lines.tolist()) + '\n')
        return conf
    (tmp_path / 'train.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())))
    (tmp_path / 'test.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())))
    if 'raw_u1' in g:
        (tmp_path / 'trust.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
            g['raw_u1'].tolist(), g['raw_u2'].tolist(), g['raw_w'].tolist())))
    return (conf.replace('./dataset/FilmTrust/trainset.txt', 'train.txt')
            .replace('./dataset/FilmTrust/testset.txt', 'test.txt').replace('./dataset/FilmTrust/trust.txt', 'trust.txt'))


def _execute(g, tmp_path, monkeypatch, conf_text):
    """Runs the configuration through QRec's data loading and the drop-in's execute: (model, epoch lines)."""
    from qrec_b200.QRec import QRec, _model_class
    from qrec_b200.util.config import ModelConf
    monkeypatch.chdir(tmp_path)
    (tmp_path / 'run.conf').write_text(conf_text)
    random.seed(int(g['seed']))
    np.random.seed(int(g['seed']))
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        q = QRec(ModelConf('run.conf'))
        cls = _model_class(q.config['model.name'])
        model = (cls(q.config, q.trainingData, q.testData, q.relation) if q.config.contains('social')
                 else cls(q.config, q.trainingData, q.testData))
        model.execute()
    lines = [ln for ln in out.getvalue().splitlines() if ' epoch ' in ln and 'loss = ' in ln]
    return model, lines


def _check_dropin(g, tmp_path, monkeypatch, case):
    model, lines = _execute(g, tmp_path, monkeypatch, _write_inputs(g, tmp_path, str(g['conf']), case))
    assert [m.strip() for m in model.measure] == g['measure'].tolist()
    assert lines == g['epoch_lines'].tolist()
    return model


@pytest.mark.parametrize('name', ['EE', 'SREE'])
def test_qrec_execute_reproduces_the_reference_filmtrust_run(torch, name, tmp_path, monkeypatch):
    g = film(name)
    model = _check_dropin(g, tmp_path, monkeypatch, False)
    assert [e[3] for e in model.data.testData] == g['test_pred'].tolist()
    for k in ('P', 'Q', 'Bu', 'Bi'):
        np.testing.assert_allclose(getattr(model, k), g[k + '_last'], rtol=1e-10, atol=1e-12)
    assert model.device_tables() is None


@pytest.mark.parametrize('tag', TAGS)
def test_qrec_execute_reproduces_the_constructed_runs(torch, tag, tmp_path, monkeypatch):
    _check_dropin(cases()[tag], tmp_path, monkeypatch, True)


def _rec_items(line):
    return line.split(':')[0] + ':' + ''.join(' ' + a + b for a, b in re.findall(r'\(([^,]+),[^)]*\)(\*?)', line))


def test_sree_ranking_run_recommends_the_reference_items(torch, tmp_path, monkeypatch):
    """item.ranking=on -topN 10: the same epoch lines, ranking measure and recommended item ids (scores may differ in
    their last digits).  `-eval gpu` stays on the host ranking, with the same lists."""
    g = film('SREE')
    conf = _write_inputs(g, tmp_path, str(g['rank_conf']))
    for extra in ('', 'engine=-eval gpu\n'):
        model, lines = _execute(g, tmp_path, monkeypatch, conf + extra)
        assert lines == g['rank_epoch_lines'].tolist()
        assert [m.strip() for m in model.measure] == g['rank_measure'].tolist()
        assert [_rec_items(ln) for ln in model.recOutput[1:]] == g['rank_rec_items'].tolist()


@pytest.mark.parametrize('name', ['EE', 'SREE'])
def test_f32_and_fast_mode_land_near_the_reference(torch, name, tmp_path, monkeypatch):
    g = film(name)
    conf = _write_inputs(g, tmp_path, str(g['conf']))
    for extra in ('engine=-precision f32\n', 'engine=-mode fast\n'):
        model, _ = _execute(g, tmp_path, monkeypatch, conf + extra)
        assert model.P.dtype == np.float64
        for got, ref in zip(model.measure, g['measure'].tolist()):
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-3


SHIPPED = {  # config/EE.conf and config/SREE.conf as QRec ships them
    'EE': ('ratings=./dataset/FilmTrust/ratings.txt\nratings.setup=-columns 0 1 2\nmodel.name=EE\n'
           'evaluation.setup=-ap 0.2 -tf\nitem.ranking=off -topN 10\nnum.factors=10\nnum.max.epoch=100\n'
           'batch_size=3000\nlearnRate=-init 0.005 -max 1\nreg.lambda=-u 0.005 -i 0.005 -b 0.005 -s 0.1\n'
           'output.setup=on -dir ./results/\n'),
    'SREE': ('ratings=./dataset/FilmTrust/trainset.txt\nsocial=./dataset/FilmTrust/trust.txt\n'
             'ratings.setup=-columns 0 1 2\nsocial.setup=-columns 0 1 2\nmodel.name=SREE\nevaluation.setup=-ap 0.3\n'
             'item.ranking=on -topN 10\nnum.factors=10\nnum.max.epoch=20\nlearnRate=-init 0.01 -max 1\n'
             'reg.lambda=-u 0.01 -i 0.01 -b 0.01 -s 0.1\nSREE=-alpha 0.5\noutput.setup=on -dir ./results/\n')}


@pytest.mark.parametrize('name', ['EE', 'SREE'])
def test_python_m_qrec_b200_runs_the_shipped_conf(torch, name, tmp_path, monkeypatch, capsys):
    """The shipped configurations from files on disk, every epoch.  EE.conf sets `-tf`: the drop-in warns and runs
    trainModel, as the engine's BasicMF and PMF do."""
    g = film('SREE')
    monkeypatch.chdir(tmp_path)
    os.makedirs('dataset/FilmTrust')
    with gzip.open(os.path.join(GOLD, 'filmtrust_ratings.txt.gz'), 'rb') as src:
        with open('dataset/FilmTrust/ratings.txt', 'wb') as dst:
            dst.write(src.read())
    for fname, cols in (('trainset.txt', ('train_users', 'train_items', 'train_rating')),
                        ('trust.txt', ('raw_u1', 'raw_u2', 'raw_w'))):
        with open('dataset/FilmTrust/' + fname, 'w') as f:
            for x in zip(*(g[c].tolist() for c in cols)):
                f.write('%s %s %s\n' % x)
    with open(name + '.conf', 'w') as f:
        f.write(SHIPPED[name])
    from qrec_b200.__main__ import main
    measure = main([name + '.conf', '--seed', '11'])
    out = capsys.readouterr().out
    lines = [ln for ln in out.splitlines() if ' epoch ' in ln and 'loss = ' in ln]
    epochs = 100 if name == 'EE' else 20
    assert len(lines) == epochs and ('epoch %d:' % epochs) in lines[-1]
    assert ('WARNING: EE has no trainModel_tf; `-tf` ignored, running trainModel().' in out) == (name == 'EE')
    values = [float(m.strip().split(':')[1]) for m in measure if ':' in m]
    assert values and all(np.isfinite(values))
    if name == 'EE':
        assert 0.5 < values[0] < 1.0                       # MAE on the 20 % split
    else:
        assert measure[0].strip() == 'Top 10'
