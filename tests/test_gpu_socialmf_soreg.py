"""SocialMF (K9 kind 4 + K17 kind 0) and SoReg (K9 kind 1 + K17 kind 1, device Pearson similarities) on the GPU
against the reference's golden runs and the numpy oracle."""
import contextlib
import io
import os
import random
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import knn_oracle as KO                 # noqa: E402
from oracle import socialmf_soreg_oracle as SM      # noqa: E402
from oracle import sorec_rste_oracle as SR          # noqa: E402
from test_social_rating_cpu import _d, conf_value, orders          # noqa: E402
from test_socialmf_soreg_cpu import (TAGS, _csr, _random_graph, case_files, cases, film, load_run, social_lists,  # noqa: E402
                                     wrapper_cases)

pytestmark = pytest.mark.gpu
KIND = {'SocialMF': 0, 'SoReg': 1}


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _lists_csr(lists):
    rowptr, cols = _csr([ids for ids, _ in lists])
    vals = np.array([v for _, vs in lists for v in vs], np.float64)
    return rowptr, cols, vals


class Pass(object):
    """The user pass of one model through the engine wrappers, on device tables of one dtype."""

    def __init__(self, torch, E, name, U, visit, fl, gl, dtype):
        self.t, self.E, self.kind, self.dt = torch, E, KIND[name], dtype
        fr, fc, fv = _lists_csr(fl)
        gr, gc, gv = _lists_csr(gl)
        visit = np.asarray(visit, np.int32)
        pos, self.depth = E.social_order_prepare(visit, U, fr, fc, gr, gc)
        i = lambda a: torch.from_numpy(a).cuda()                            # noqa: E731
        v = lambda a: torch.from_numpy(a).to('cuda', dtype)                 # noqa: E731
        self.args = (i(visit), i(pos), i(fr), i(fc), v(fv), i(gr), i(gc), v(gv) if self.kind == 1 else None)

    def __call__(self, P, lr, coef, n_warps=0):
        loss = self.t.zeros(1, dtype=self.t.float64, device='cuda')
        self.E.social_user_pass(self.kind, P, *self.args, lr, coef, loss, n_warps=n_warps)
        return float(loss.item())


def _coef(g, name):
    return conf_value(g, 'reg.lambda', '-s') if name == 'SocialMF' else conf_value(g, 'SoReg', '-alpha')


def _replay_on_device(torch, E, g, name, dtype=None):
    """Both passes of every recorded epoch on the device (float64).  After each rating pass the user pass also runs
    in the oracle on the same input rows, and the two must agree bit for bit.  Returns (P, Q after epoch 1, after the
    last epoch, losses)."""
    dtype = dtype or torch.float64
    users, items, _, _, _, u0, i0 = load_run(g)
    U, I = len(users), len(items)
    visit, fl, gl = social_lists(g, name)
    sp = Pass(torch, E, name, U, visit, fl, gl, dtype)
    P, Q = (torch.from_numpy(t).to('cuda', dtype) for t in SR.initial_tables(int(g['seed']), U, I, _d(g), False))
    reg_u, reg_i, coef = conf_value(g, 'reg.lambda', '-u'), conf_value(g, 'reg.lambda', '-i'), _coef(g, name)
    losses, first = [], None
    for e, o in enumerate(orders(g)):
        lr = float(g['lrate'][e][0])
        u, i, r = u0[o], i0[o], g['train_rating'][o]
        wu, wi = E.mf_order_prepare(u, i, U, I)
        loss = torch.zeros(1, dtype=torch.float64, device='cuda')
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
        E.mf_sgd_ordered(E.SOCIALMF_RATINGS if name == 'SocialMF' else 1, P, Q, d(u), d(i), d(r).to(dtype), d(wu),
                         d(wi), lr, reg_u, reg_i, loss)
        Ph = P.cpu().numpy().copy()
        social = sp(P, lr, coef)
        if name == 'SocialMF':
            want = SM.socialmf_user_pass(Ph, visit, fl, lr, coef)
        else:
            want = SM.soreg_user_pass(Ph, visit, fl, gl, lr, coef)
        assert np.array_equal(P.cpu().numpy(), Ph), 'user pass != oracle, epoch %d' % (e + 1)
        assert abs(social - float(want)) <= 1e-12 * max(1.0, abs(float(want)))
        Pn, Qn = P.double().cpu().numpy(), Q.double().cpu().numpy()
        losses.append(float(loss.item()) + social + (reg_u * (Pn * Pn).sum() + reg_i * (Qn * Qn).sum()))
        if e == 0:
            first = (Pn.copy(), Qn.copy())
    return first, (P.double().cpu().numpy(), Q.double().cpu().numpy()), losses


def _check_f64(torch, E, g, name):
    first, last, losses = _replay_on_device(torch, E, g, name)
    # the rating pass's dot product is a warp tree sum (K9), not numpy's sequential one: the tables agree to rounding
    for t, k in zip(first, 'PQ'):
        np.testing.assert_allclose(t.astype(np.float32), g[k + '_epoch1'], rtol=1e-6, atol=1e-7)
    for t, k in zip(last, 'PQ'):
        np.testing.assert_allclose(t, g[k + '_last'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(losses, g['loss'], rtol=1e-12)


@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
def test_f64_kernels_reproduce_the_reference_filmtrust_run(torch, E, name):
    _check_f64(torch, E, film(name), name)


@pytest.mark.parametrize('tag', TAGS)
def test_f64_kernels_reproduce_the_constructed_runs(torch, E, tag):
    _check_f64(torch, E, cases()[tag], 'SoReg' if tag.startswith('soreg') else 'SocialMF')


@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
def test_f32_kernels_match_the_f32_oracle(torch, E, name):
    g = film(name)
    users, items, _, _, _, u0, i0 = load_run(g)
    visit, fl, gl = social_lists(g, name)
    U, I = len(users), len(items)
    P0, Q0 = (t.astype(np.float32) for t in SR.initial_tables(int(g['seed']), U, I, _d(g), False))
    o = orders(g)[1]
    lr, reg_u, reg_i, coef = float(g['lrate'][0][0]), conf_value(g, 'reg.lambda', '-u'), conf_value(
        g, 'reg.lambda', '-i'), _coef(g, name)
    P, Q = torch.from_numpy(P0.copy()).cuda(), torch.from_numpy(Q0.copy()).cuda()
    u, i, r = u0[o], i0[o], g['train_rating'][o]
    wu, wi = E.mf_order_prepare(u, i, U, I)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.mf_sgd_ordered(E.SOCIALMF_RATINGS if name == 'SocialMF' else 1, P, Q, d(u), d(i), d(r).float(), d(wu), d(wi),
                     lr, reg_u, reg_i, loss)
    Pass(torch, E, name, U, visit, fl, gl, torch.float32)(P, lr, coef)
    Ph, Qh = P0.copy(), Q0.copy()
    if name == 'SocialMF':
        SM.socialmf_epoch(Ph, Qh, u, i, r, visit, fl, lr, reg_u, reg_i, coef)
    else:
        SM.soreg_epoch(Ph, Qh, u, i, r, visit, fl, gl, lr, reg_u, reg_i, coef)
    np.testing.assert_allclose(P.cpu().numpy(), Ph, rtol=2e-4, atol=2e-6)
    np.testing.assert_allclose(Q.cpu().numpy(), Qh, rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
@pytest.mark.parametrize('d', [1, 33, 64, 256])
def test_result_does_not_depend_on_the_grid(torch, E, name, dtype, d):
    """A dense trust graph (up to 24 followees per user, a self-follow, zero weights, negative similarities) and a
    visiting order that skips some users: n_warps 1 (one CTA of 8 warps), 64 and the default give the same bits,
    and the bits of the sequential oracle in the same precision."""
    U = 200
    rs = np.random.RandomState(d)
    followees, followers = _random_graph(rs, U, 24)
    vals = {(a, b): float(np.round(rs.randn(), 3)) for a in range(U) for b in followees[a]}
    for b in followees[2]:
        vals[(2, b)] = 0.0                                                 # SocialMF's denom == 0
    fl = [(followees[a], [vals[(a, b)] for b in followees[a]]) for a in range(U)]
    gl = [(followers[b], [vals[(a, b)] for a in followers[b]]) for b in range(U)]
    visit = [int(x) for x in rs.permutation(U)[:180]]
    dt = getattr(torch, dtype)
    npdt = np.float64 if dtype == 'float64' else np.float32
    P0 = (rs.rand(U, d) / 3).astype(npdt)
    sp = Pass(torch, E, name, U, visit, fl, gl, dt)
    out = []
    for n_warps in (1, 64, 0):
        P = torch.from_numpy(P0.copy()).cuda()
        loss = sp(P, 0.05, 0.1, n_warps=n_warps)
        out.append((P.cpu().numpy(), loss))
    for P, loss in out[1:]:
        assert np.array_equal(P, out[0][0])
        assert abs(loss - out[0][1]) <= 1e-12 * abs(out[0][1])
    Ph = P0.copy()
    want = (SM.socialmf_user_pass(Ph, visit, fl, 0.05, 0.1) if name == 'SocialMF'
            else SM.soreg_user_pass(Ph, visit, fl, gl, 0.05, 0.1))
    assert np.array_equal(out[0][0], Ph)
    assert abs(out[0][1] - float(want)) <= (1e-12 if dtype == 'float64' else 1e-5) * abs(float(want))
    assert sp.depth == SM.schedule(visit, U, followees, followers)[1]


# ------------------------------------------------------------------------------------------------ similarities
def _pair_sims(torch, E, rows_by_id, pairs, weights):
    """knn_pair_similarity over id-keyed rows {row id: {col: value}} (insertion order)."""
    n = len(rows_by_id)
    rowptr = np.zeros(n + 1, np.int64)
    rowptr[1:] = np.cumsum([len(rows_by_id[k]) for k in range(n)])
    cols = np.array([c for k in range(n) for c in rows_by_id[k]], np.int32)
    vals = np.array([v for k in range(n) for v in rows_by_id[k].values()], np.float64)
    means = np.array([sum(rows_by_id[k].values()) / len(rows_by_id[k]) for k in range(n)], np.float64)
    sq = E.knn_squares(rowptr, vals, means, 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    scols, svals = E.knn_sorted_view(t(rowptr), t(cols), t(vals))
    _, ssq = E.knn_sorted_view(t(rowptr), t(cols), t(sq))
    a = np.array([p[0] for p in pairs], np.int32)
    b = np.array([p[1] for p in pairs], np.int32)
    return E.knn_pair_similarity(t(rowptr), t(cols), t(vals), t(sq), t(means), scols, svals, ssq, t(a), t(b),
                                 t(np.asarray(weights, np.float64))).cpu().numpy()


def test_pair_similarity_equals_the_recorded_filmtrust_sim(torch, E):
    g = film('SoReg')
    users, items, followees, _, rows, _, _ = load_run(g)
    names = g['user_names'].tolist()
    _, pairs = SM.soreg_similarities(names, followees, rows)
    by_id = {users[n]: {items[i]: v for i, v in rows[n].items()} for n in names}
    got = _pair_sims(torch, E, by_id, [(users[a], users[b]) for a, b in pairs],
                     [followees[a][b] for a, b in pairs])
    rec = {(a, b): v for a, b, v in zip(g['sim_user'].tolist(), g['sim_friend'].tolist(), g['sim_value'].tolist())}
    want = np.array([rec[p] for p in pairs])
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    assert len(pairs) > 1000


def test_pair_similarity_equals_pearson_sp_on_random_rows(torch, E):
    """Rows with repeated values, a constant row (zero variance), rows sharing one key, rows sharing none, and a
    row paired with itself."""
    rs = np.random.RandomState(3)
    rows = {}
    for k in range(60):
        keys = rs.choice(40, size=rs.randint(1, 15), replace=False).tolist()
        rows[k] = {c: float(rs.randint(1, 9) * 0.5) for c in keys}
    rows[0] = {c: 3.0 for c in (1, 5, 9, 13)}                              # zero variance
    rows[1] = {100: 2.0, 5: 4.0}                                           # shares one key with row 0
    rows[2] = {200 + c: 1.5 * c for c in range(5)}                         # shares nothing
    pairs = [(int(rs.randint(60)), int(rs.randint(60))) for _ in range(400)] + [(0, 1), (1, 0), (2, 3), (0, 4),
                                                                                  (5, 5), (0, 0)]
    w = np.round(rs.rand(len(pairs)), 2)
    got = _pair_sims(torch, E, rows, pairs, w)
    want = np.array([(KO.similarity(rows[a], rows[b], 'pcc') + float(x)) / 2.0 for (a, b), x in zip(pairs, w)])
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


def test_wrappers_raise_qrecerror_on_each_invalid_input(torch, E):
    """The valid calls run; every invalid input, shapes and contents alike, raises its own QRecError."""
    pass_ok, sim_ok, bad = wrapper_cases(torch, 'cuda')
    E.social_user_pass(**pass_ok)
    E.knn_pair_similarity(**sim_ok)
    torch.cuda.synchronize()
    assert float(pass_ok['loss'].item()) > 0
    for k, (call, message, _) in enumerate(bad):
        with pytest.raises(E.QRecError, match=message):
            call()
            pytest.fail('case %d did not raise' % k)


# ------------------------------------------------------------------------------------------------ drop-ins
def _write_inputs(g, tmp_path, case=False):
    if case:
        for name, lines in case_files().items():
            (tmp_path / name).write_text('\n'.join(lines.tolist()) + '\n')
        return str(g['conf'])
    (tmp_path / 'train.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())))
    (tmp_path / 'test.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())))
    (tmp_path / 'trust.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['raw_u1'].tolist(), g['raw_u2'].tolist(), g['raw_w'].tolist())))
    return (str(g['conf']).replace('./dataset/FilmTrust/trainset.txt', 'train.txt')
            .replace('./dataset/FilmTrust/testset.txt', 'test.txt').replace('./dataset/FilmTrust/trust.txt', 'trust.txt'))


def _execute(g, tmp_path, monkeypatch, conf_text, extra=''):
    from qrec_b200.QRec import QRec
    from qrec_b200.util.config import ModelConf
    monkeypatch.chdir(tmp_path)
    (tmp_path / 'run.conf').write_text(conf_text + extra)
    random.seed(int(g['seed']))
    np.random.seed(int(g['seed']))
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        measure = QRec(ModelConf('run.conf')).execute()
    lines = [ln for ln in out.getvalue().splitlines() if ' epoch ' in ln and 'loss = ' in ln]
    return [m.strip() for m in measure], lines, out.getvalue()


def _check_dropin(g, tmp_path, monkeypatch, case):
    measure, lines, out = _execute(g, tmp_path, monkeypatch, _write_inputs(g, tmp_path, case))
    assert measure == g['measure'].tolist()
    assert lines == g['epoch_lines'].tolist()
    return out


@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
def test_qrec_execute_reproduces_the_reference_filmtrust_run(torch, name, tmp_path, monkeypatch):
    out = _check_dropin(film(name), tmp_path, monkeypatch, False)
    assert ('constructing similarity matrix...' in out) == (name == 'SoReg')


@pytest.mark.parametrize('tag', TAGS)
def test_qrec_execute_reproduces_the_constructed_runs(torch, tag, tmp_path, monkeypatch):
    _check_dropin(cases()[tag], tmp_path, monkeypatch, True)


def test_dropin_predictions_and_similarities(torch, tmp_path, monkeypatch):
    """The drop-in's test predictions are the reference's, and SoReg's Sim dict is the recorded one bit for bit."""
    from qrec_b200.model.rating.SoReg import SoReg
    from qrec_b200.QRec import QRec
    from qrec_b200.util.config import ModelConf
    g = film('SoReg')
    monkeypatch.chdir(tmp_path)
    (tmp_path / 'run.conf').write_text(_write_inputs(g, tmp_path))
    random.seed(int(g['seed']))
    np.random.seed(int(g['seed']))
    with contextlib.redirect_stdout(io.StringIO()):
        q = QRec(ModelConf('run.conf'))
        model = SoReg(q.config, q.trainingData, q.testData, q.relation)
        model.execute()
    got = [(a, b, v) for a in model.Sim for b, v in model.Sim[a].items()]
    rec = list(zip(g['sim_user'].tolist(), g['sim_friend'].tolist(), g['sim_value'].tolist()))
    assert sorted(got) == sorted(rec)
    assert [e[3] for e in model.data.testData] == g['test_pred'].tolist()
    np.testing.assert_allclose(model.P, g['P_last'], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
def test_f32_and_fast_mode_land_near_the_reference(torch, name, tmp_path, monkeypatch):
    g = film(name)
    conf = _write_inputs(g, tmp_path)
    for extra in ('engine=-precision f32\n', 'engine=-mode fast\n'):
        measure, _, _ = _execute(g, tmp_path, monkeypatch, conf, extra)
        for got, ref in zip(measure, g['measure'].tolist()):
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-3


SHIPPED = {  # config/SocialMF.conf and config/SoReg.conf as QRec ships them
    'SocialMF': dict(topn=30, d=5, regs='-u 0.05 -i 0.05 -b 0.1 -s 0.1', extra=''),
    'SoReg': dict(topn=10, d=10, regs='-u 0.02 -i 0.02 -b 0.1 -s 0.02', extra='SoReg=-alpha 0.1\n')}


@pytest.mark.parametrize('name', ['SocialMF', 'SoReg'])
def test_python_m_qrec_b200_runs_the_shipped_conf(torch, name, tmp_path, monkeypatch, capsys):
    """The shipped configurations, 30 epochs, from files on disk.  SocialMF ends where the unmodified reference ends
    (seed 11: MAE 0.623975386376645, RMSE 0.8307707626674363).  SoReg at the shipped settings diverges in epoch 4 in
    the reference too: its first three epochs print the reference's lines, then the run stops with the NaN message
    and exit code -1, as the reference's does."""
    g = film(name)
    monkeypatch.chdir(tmp_path)
    os.makedirs('dataset/FilmTrust')
    for fname, cols in (('trainset.txt', ('train_users', 'train_items', 'train_rating')),
                        ('testset.txt', ('test_users', 'test_items', 'test_rating')),
                        ('trust.txt', ('raw_u1', 'raw_u2', 'raw_w'))):
        with open('dataset/FilmTrust/' + fname, 'w') as f:
            for x in zip(*(g[c].tolist() for c in cols)):
                f.write('%s %s %s\n' % x)
    s = SHIPPED[name]
    with open(name + '.conf', 'w') as f:
        f.write('ratings=./dataset/FilmTrust/trainset.txt\nsocial=./dataset/FilmTrust/trust.txt\n'
                'ratings.setup=-columns 0 1 2\nsocial.setup=-columns 0 1 2\nmodel.name=%s\n'
                'evaluation.setup=-testSet ./dataset/FilmTrust/testset.txt\nitem.ranking=off -topN %d\n'
                'num.factors=%d\nnum.max.epoch=30\nlearnRate=-init 0.05 -max 1\nreg.lambda=%s\n%s'
                'output.setup=on -dir ./results/\n' % (name, s['topn'], s['d'], s['regs'], s['extra']))
    from qrec_b200.__main__ import main
    argv = [name + '.conf', '--seed', str(int(g['seed']))]
    if name == 'SoReg':
        with pytest.raises(SystemExit) as stop:
            main(argv)
        assert stop.value.code == -1
        out = capsys.readouterr().out
        lines = [ln for ln in out.splitlines() if ' epoch ' in ln and 'loss = ' in ln]
        assert lines == g['epoch_lines'].tolist()
        assert 'Loss = NaN or Infinity' in out
        return
    measure = main(argv)
    out = capsys.readouterr().out
    assert 'Running time:' in out and 'epoch 30:' in out
    mae, rmse = (float(m.strip().split(':')[1]) for m in measure[:2])
    assert abs(mae - 0.623975386376645) < 1e-6 and abs(rmse - 0.8307707626674363) < 1e-6
