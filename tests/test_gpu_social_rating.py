"""SoRec (K9 kind 3) and RSTE (K16) on the GPU against the reference's golden runs and the numpy oracle."""
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
from oracle import sorec_rste_oracle as SR               # noqa: E402
from test_social_rating_cpu import (_d, cases, conf_value, film, load_run, orders, wrapper_cases)   # noqa: E402

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


def _csr(fl, U):
    rowptr = np.zeros(U + 1, np.int64)
    rowptr[1:] = np.cumsum([len(ids) for ids, _ in fl])
    cols = np.concatenate([ids for ids, _ in fl] + [np.zeros(0)]).astype(np.int32)
    w = np.concatenate([np.asarray(ws, np.float64) for _, ws in fl] + [np.zeros(0)])
    denom = np.array([ws.sum() if len(ws) else 0.0 for _, ws in fl], np.float64)
    return rowptr, cols, w, denom


class Engine(object):
    """The two models' epochs through the engine wrappers, on device tables of one dtype."""

    def __init__(self, torch, E, dtype, U, I, fl=None, edges=None):
        self.t, self.E, self.dt, self.U, self.I = torch, E, dtype, U, I
        dev = torch.device('cuda')
        self.dev = dev
        if fl is not None:
            rowptr, cols, w, denom = _csr(fl, U)
            self.rowptr, self.cols = rowptr, cols
            self.social = (torch.from_numpy(rowptr).to(dev), torch.from_numpy(cols).to(dev),
                           torch.from_numpy(w).to(dev, dtype), torch.from_numpy(denom).to(dev, dtype))
        if edges is not None:
            eu, ev, et = edges
            wu, wv = E.mf_order_prepare(eu, ev, U, U)
            self.edges = [torch.from_numpy(np.asarray(a)).to(dev) for a in (eu, ev, wu, wv)]
            self.et = torch.tensor(np.asarray(et, np.float64), device=dev, dtype=dtype)

    def up(self, a):
        return self.t.from_numpy(np.ascontiguousarray(a)).to(self.dev, self.dt).contiguous()

    def rste(self, P, Q, u, i, r, lr, reg_u, reg_i, alpha, n_warps=0):
        t, E = self.t, self.E
        wu, wi, wr, pr, pos, depth = E.rste_order_prepare(u, i, self.U, self.I, self.rowptr, self.cols)
        loss = t.zeros(1, dtype=t.float64, device=self.dev)
        dv = [t.from_numpy(a).to(self.dev) for a in (u, i, wu, wi, wr, pr, pos)]
        E.rste_sgd_ordered(P, Q, dv[0], dv[1], self.up(r), dv[2], dv[3], dv[4], dv[5], dv[6], *self.social, lr, reg_u,
                           reg_i, alpha, loss, n_warps=n_warps)
        return float(loss.item())

    def sorec(self, P, Q, Z, u, i, r, lr, reg_u, reg_i, reg_s, reg_z, n_warps=0):
        t, E = self.t, self.E
        wu, wi = E.mf_order_prepare(u, i, self.U, self.I)
        loss = t.zeros(2, dtype=t.float64, device=self.dev)
        dv = [t.from_numpy(a).to(self.dev) for a in (u, i, wu, wi)]
        E.mf_sgd_ordered(1, P, Q, dv[0], dv[1], self.up(r), dv[2], dv[3], lr, reg_u, reg_i, loss[0:1], n_warps=n_warps)
        e = self.edges
        E.mf_sgd_ordered(E.SOREC_EDGES, P, Z, e[0], e[1], self.et, e[2], e[3], lr, reg_s, reg_z, loss[1:2],
                         n_warps=n_warps)
        return float(loss.sum().item())


def _film_engine(torch, E, g, name, dtype):
    users, items, rel, followees, followers, u0, i0 = load_run(g)
    fl = SR.followee_lists(g['user_names'].tolist(), users, followees)
    edges = SR.sorec_edges(users, followees, followers, rel) if name == 'SoRec' else None
    eng = Engine(torch, E, dtype, len(users), len(items), fl=fl, edges=edges)
    tables = [eng.up(t) for t in SR.initial_tables(int(g['seed']), len(users), len(items), _d(g), name == 'SoRec')]
    return eng, tables, u0, i0, fl, edges


def _regs(g, name):
    if name == 'SoRec':
        return (conf_value(g, 'reg.lambda', '-u'), conf_value(g, 'reg.lambda', '-i'), conf_value(g, 'reg.lambda', '-s'),
                conf_value(g, 'SoRec', '-z'))
    return conf_value(g, 'reg.lambda', '-u'), conf_value(g, 'reg.lambda', '-i'), conf_value(g, 'RSTE', '-alpha')


@pytest.mark.parametrize('name', ['SoRec', 'RSTE'])
def test_f64_kernels_reproduce_the_reference_over_three_epochs(torch, E, name):
    g = film(name)
    eng, tables, u0, i0, _, _ = _film_engine(torch, E, g, name, torch.float64)
    regs = _regs(g, name)
    losses = []
    for e, o in enumerate(orders(g)):
        lr = float(g['lrate'][e][0])
        if name == 'SoRec':
            sq = eng.sorec(*tables, u0[o], i0[o], g['train_rating'][o], lr, *regs)
            P, Q, Z = (t.cpu().numpy() for t in tables)
            losses.append(sq + (regs[0] * (P * P).sum() + regs[1] * (Q * Q).sum() + regs[3] * (Z * Z).sum()))
        else:
            sq = eng.rste(*tables, u0[o], i0[o], g['train_rating'][o], lr, *regs)
            P, Q = (t.cpu().numpy() for t in tables)
            losses.append(sq + (regs[0] * (P * P).sum() + regs[1] * (Q * Q).sum()))
        if e == 0:
            for t, k in zip(tables, 'PQZ'):
                np.testing.assert_allclose(t.cpu().numpy(), g[k + '_epoch1'], rtol=1e-6, atol=1e-7)
    for t, k in zip(tables, 'PQZ'):
        np.testing.assert_allclose(t.cpu().numpy(), g[k + '_last'], rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(losses, g['loss'], rtol=1e-9)


@pytest.mark.parametrize('name', ['SoRec', 'RSTE'])
def test_f32_kernels_match_the_f32_oracle(torch, E, name):
    g = film(name)
    eng, tables, u0, i0, fl, edges = _film_engine(torch, E, g, name, torch.float32)
    host = [t.astype(np.float32) for t in SR.initial_tables(int(g['seed']), eng.U, eng.I, _d(g), name == 'SoRec')]
    regs = _regs(g, name)
    o = orders(g)[1]                                                  # a shuffled epoch
    lr = float(g['lrate'][0][0])
    if name == 'SoRec':
        eng.sorec(*tables, u0[o], i0[o], g['train_rating'][o], lr, *regs)
        SR.sorec_epoch(*host, u0[o], i0[o], g['train_rating'][o], *edges, lr, *regs)
    else:
        eng.rste(*tables, u0[o], i0[o], g['train_rating'][o], lr, *regs)
        SR.rste_epoch(*host, u0[o], i0[o], g['train_rating'][o], fl, lr, *regs)
    for t, h in zip(tables, host):
        np.testing.assert_allclose(t.cpu().numpy(), h, rtol=2e-4, atol=2e-6)


def _synthetic(U, I, n, max_deg, seed):
    rs = np.random.RandomState(seed)
    fl = []
    for a in range(U):
        deg = rs.randint(0, max_deg + 1)
        ids = rs.choice(U, size=min(deg, U), replace=False)
        fl.append((ids.astype(np.int64), np.round(rs.rand(len(ids)), 2)))
    fl[3] = (np.array([3, 1], np.int64), np.array([0.5, 0.25]))         # a self-follow
    fl[4] = (np.array([5, 6], np.int64), np.array([0.0, 0.0]))          # denom == 0
    fl[5] = (np.zeros(0, np.int64), np.zeros(0))                        # follows nobody
    u = rs.randint(0, U, size=n).astype(np.int32)
    i = rs.randint(0, I, size=n).astype(np.int32)
    r = (rs.randint(1, 9, size=n) * 0.5).astype(np.float64)
    return fl, u, i, r


@pytest.mark.parametrize('d', [1, 5, 31, 32, 33, 64, 65, 128, 256])
def test_every_lane_shape_matches_the_f64_oracle(torch, E, d):
    U, I, n = 50, 30, 800
    fl, u, i, r = _synthetic(U, I, n, 8, d)
    rs = np.random.RandomState(100 + d)
    P0, Q0, Z0 = rs.rand(U, d) / 3, rs.rand(I, d) / 3, rs.rand(U, d) / 10
    # RSTE
    eng = Engine(torch, E, torch.float64, U, I, fl=fl)
    P, Q = eng.up(P0), eng.up(Q0)
    sq = eng.rste(P, Q, u, i, r, 0.01, 0.001, 0.002, 0.6)
    Ph, Qh = P0.copy(), Q0.copy()
    ref = SR.rste_epoch(Ph, Qh, u, i, r, fl, 0.01, 0.001, 0.002, 0.6) - (0.001 * (Ph * Ph).sum() + 0.002 * (Qh * Qh).sum())
    np.testing.assert_allclose(P.cpu().numpy(), Ph, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(Q.cpu().numpy(), Qh, rtol=1e-9, atol=1e-12)
    assert abs(sq - ref) <= 1e-9 * abs(ref)
    # SoRec's two passes, the edges being every (u, f) of the followee lists in order
    eu = np.array([a for a in range(U) for _ in fl[a][0]], np.int32)
    ev = np.concatenate([ids for ids, _ in fl]).astype(np.int32)
    et = np.concatenate([w for _, w in fl]).tolist()
    eng = Engine(torch, E, torch.float64, U, I, edges=(eu, ev, et))
    P, Q, Z = eng.up(P0), eng.up(Q0), eng.up(Z0)
    eng.sorec(P, Q, Z, u, i, r, 0.01, 0.05, 0.05, 0.1, 0.1)
    Ph, Qh, Zh = P0.copy(), Q0.copy(), Z0.copy()
    SR.sorec_epoch(Ph, Qh, Zh, u, i, r, eu, ev, et, 0.01, 0.05, 0.05, 0.1, 0.1)
    for t, h in ((P, Ph), (Q, Qh), (Z, Zh)):
        np.testing.assert_allclose(t.cpu().numpy(), h, rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_result_does_not_depend_on_the_grid_on_a_dense_trust_graph(torch, E, dtype):
    """Each user follows up to half of the 64 users (a quarter on average): every row is read by many followers
    between its writes.  n_warps=1 starts one CTA of 8 warps; it and a full grid give the same bits, and both equal
    the sequential oracle in the same precision."""
    U, I, n, d = 64, 40, 4000, 33
    fl, u, i, r = _synthetic(U, I, n, 32, 7)
    dt = getattr(torch, dtype)
    npdt = np.float64 if dtype == 'float64' else np.float32
    tol = dict(rtol=1e-9, atol=1e-12) if dtype == 'float64' else dict(rtol=2e-4, atol=2e-6)
    rs = np.random.RandomState(8)
    P0, Q0 = rs.rand(U, d) / 3, rs.rand(I, d) / 3
    out = []
    for n_warps in (1, 0):
        eng = Engine(torch, E, dt, U, I, fl=fl)
        P, Q = eng.up(P0), eng.up(Q0)
        loss = eng.rste(P, Q, u, i, r, 0.01, 0.001, 0.001, 0.6, n_warps=n_warps)
        out.append((P.cpu().numpy(), Q.cpu().numpy(), loss))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    assert abs(out[0][2] - out[1][2]) <= 1e-12 * abs(out[0][2])       # per-warp partials, added in any order
    Ph, Qh = P0.astype(npdt), Q0.astype(npdt)
    ref = SR.rste_epoch(Ph, Qh, u, i, r, fl, 0.01, 0.001, 0.001, 0.6) - float(0.001 * (Ph * Ph).sum() + 0.001 * (Qh * Qh).sum())
    np.testing.assert_allclose(out[0][0], Ph, **tol)
    np.testing.assert_allclose(out[0][1], Qh, **tol)
    assert abs(out[0][2] - ref) <= (1e-9 if dtype == 'float64' else 1e-4) * abs(ref)
    eu = np.array([a for a in range(U) for _ in fl[a][0]], np.int32)
    ev = np.concatenate([ids for ids, _ in fl]).astype(np.int32)
    et = np.concatenate([w for _, w in fl]).tolist()
    res = []
    for n_warps in (1, 0):
        eng = Engine(torch, E, dt, U, I, edges=(eu, ev, et))
        P, Q, Z = eng.up(P0), eng.up(Q0), eng.up(P0[::-1])
        eng.sorec(P, Q, Z, u, i, r, 0.01, 0.05, 0.05, 0.1, 0.1, n_warps=n_warps)
        res.append([t.cpu().numpy() for t in (P, Q, Z)])
    assert all(np.array_equal(a, b) for a, b in zip(*res))
    host = [t.astype(npdt) for t in (P0, Q0, P0[::-1].copy())]
    SR.sorec_epoch(*host, u, i, r, eu, ev, et, 0.01, 0.05, 0.05, 0.1, 0.1)
    for got, want in zip(res[0], host):
        np.testing.assert_allclose(got, want, **tol)


def test_predict_pairs_is_the_blend(torch, E):
    U, I, d = 50, 30, 7
    fl, u, i, _ = _synthetic(U, I, 300, 8, 9)
    rs = np.random.RandomState(10)
    P0, Q0 = rs.rand(U, d), rs.rand(I, d)
    for dt, tol in ((torch.float64, 1e-12), (torch.float32, 1e-5)):
        eng = Engine(torch, E, dt, U, I, fl=fl)
        got = E.rste_predict_pairs(eng.up(P0), eng.up(Q0), torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda(),
                                   *eng.social, 0.6).double().cpu().numpy()
        want = [SR.rste_predict(P0, Q0, int(a), int(b), fl, 0.6) for a, b in zip(u, i)]
        np.testing.assert_allclose(got, want, rtol=tol)


def test_wrappers_raise_qrecerror_on_each_invalid_input(torch, E):
    """The valid calls run; every invalid input, shapes and contents alike, raises its own QRecError."""
    sgd_ok, pred_ok, edge_ok, bad = wrapper_cases(torch, 'cuda')
    E.rste_sgd_ordered(**sgd_ok)
    E.rste_predict_pairs(**pred_ok)
    E.mf_sgd_ordered(*edge_ok)
    torch.cuda.synchronize()
    assert float(sgd_ok['loss'].item()) > 0
    for k, (call, message, _) in enumerate(bad):
        with pytest.raises(E.QRecError, match=message):
            call()
            pytest.fail('case %d did not raise' % k)


# ------------------------------------------------------------------------------------------------ drop-ins
def _write_inputs(g, tmp_path, files=None):
    if files is not None:
        for name, lines in files.items():
            (tmp_path / name).write_text('\n'.join(lines.tolist()) + '\n')
        return str(g['conf'])
    (tmp_path / 'train.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist())))
    (tmp_path / 'test.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['test_users'].tolist(), g['test_items'].tolist(), g['test_rating'].tolist())))
    (tmp_path / 'trust.txt').write_text(''.join('%s %s %r\n' % x for x in zip(
        g['rel_u1'].tolist(), g['rel_u2'].tolist(), g['rel_w'].tolist())))
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
    return [m.strip() for m in measure], lines


@pytest.mark.parametrize('name', ['SoRec', 'RSTE'])
def test_qrec_execute_reproduces_the_reference_filmtrust_run(torch, name, tmp_path, monkeypatch):
    g = film(name)
    measure, lines = _execute(g, tmp_path, monkeypatch, _write_inputs(g, tmp_path))
    assert measure == g['measure'].tolist()
    assert lines == g['epoch_lines'].tolist()


@pytest.mark.parametrize('tag', ['sorec_w', 'rste_w', 'rste_rank', 'sorec_nw', 'rste_nw'])
def test_qrec_execute_reproduces_the_constructed_runs(torch, tag, tmp_path, monkeypatch):
    c = cases()
    g = c[tag]
    files = {k.split('/', 1)[1]: v for k, v in np.load(os.path.join(ROOT, 'tests', 'golden', 'social_rating_cases.npz'))
             .items() if k.startswith('files/')}
    measure, lines = _execute(g, tmp_path, monkeypatch, _write_inputs(g, tmp_path, files))
    assert measure == g['measure'].tolist()
    assert lines == g['epoch_lines'].tolist()


@pytest.mark.parametrize('name', ['SoRec', 'RSTE'])
def test_f32_and_fast_mode_land_near_the_reference(torch, name, tmp_path, monkeypatch):
    g = film(name)
    conf = _write_inputs(g, tmp_path)
    for extra in ('engine=-precision f32\n', 'engine=-mode fast\n'):
        measure, _ = _execute(g, tmp_path, monkeypatch, conf, extra)
        for got, ref in zip(measure, g['measure'].tolist()):
            assert abs(float(got.split(':')[1]) - float(ref.split(':')[1])) < 1e-3
