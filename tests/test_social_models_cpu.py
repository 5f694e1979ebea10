"""Life cycle of the social and Euclidean rating drop-ins (SoRec, RSTE, SocialMF, SoReg, EE, SREE) without a GPU: the
device is stubbed to 'cpu' and every kernel they launch is replaced by its pinned float64 oracle, so what is checked is
everything AROUND the kernels -- id mapping, the per-epoch visiting order, the trust CSRs and visiting order handed to
the user passes, loss assembly, the adaptive learning rate, the stopping rule and the evaluation -- against the
reference's recorded FilmTrust runs (tests/golden/{sorec,rste,socialmf,soreg,ee,sree}_filmtrust.npz).  The kernels
themselves are compared with the same oracles in the GPU suites."""
import contextlib
import io
import os
import random

import numpy as np
import pytest

from oracle import ee_sree_oracle as EO
from oracle import knn_oracle as KO
from oracle import socialmf_soreg_oracle as SM
from oracle import sorec_rste_oracle as SR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
LISTS = ('user_names', 'item_names', 'train_users', 'train_items', 'train_rating', 'test_users', 'test_items',
         'test_rating')
# the kernels each epoch launches, in order
EPOCH = {'SoRec': [('mf_sgd_ordered', 1), ('mf_sgd_ordered', 3)],
         'RSTE': [('rste_sgd_ordered', None), ('rste_predict_pairs', None)],
         'SocialMF': [('mf_sgd_ordered', 4), ('social_user_pass', 0)],
         'SoReg': [('mf_sgd_ordered', 1), ('social_user_pass', 1)],
         'EE': [('mf_sgd_ordered', 5)],
         'SREE': [('mf_sgd_ordered', 5), ('sree_user_pass', None)]}


def _lists(rowptr, cols, vals):
    """A CSR (tensors) as the oracles' per-row (ids, values) lists."""
    rp, c, v = rowptr.numpy().tolist(), cols.numpy(), vals.numpy()
    return [(c[a:b], v[a:b]) for a, b in zip(rp[:-1], rp[1:])]


def _edge_pass(P, Z, eu, ev, et, lr, reg_s, reg_z):
    """SoRec's trust-edge pass (K9 kind 3), the second loop of sorec_epoch: returns its loss terms."""
    loss = 0
    for uu, vv, t in zip(eu.tolist(), ev.tolist(), et.tolist()):
        euv = t - P[uu].dot(Z[vv])
        loss += reg_s * (euv ** 2)
        p, z = P[uu], Z[vv]
        P[uu] += lr * (reg_s * euv * z)
        Z[vv] += lr * (reg_s * euv * p - reg_z * z)
    return loss


def _rste_pass(P, Q, u, i, r, fl, lr, reg_u, reg_i, alpha):
    """RSTE's rating pass (K16), rste_epoch without the regulariser: returns sum e^2."""
    loss = 0
    for uu, ii, rr in zip(u.tolist(), i.tolist(), r.tolist()):
        error = rr - SR.rste_predict(P, Q, uu, ii, fl, alpha)
        loss += error ** 2
        p, q = P[uu], Q[ii]
        P[uu] += lr * (alpha * error * q - reg_u * p)
        Q[ii] += lr * (alpha * error * p - reg_i * q)
    return loss


@pytest.fixture
def calls(monkeypatch):
    """Installs the oracle engine; yields the list of (kernel, kind, n_warps) the run launched."""
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.iterativeRecommender import IterativeRecommender
    log = []

    def schedule_of(P, visit, pos, f_rowptr, f_cols, g_rowptr, g_cols):
        # the schedule handed to the kernel must describe this visiting order and these CSRs
        want, _ = E.social_order_prepare(visit.numpy(), P.shape[0], f_rowptr.numpy(), f_cols.numpy(),
                                         g_rowptr.numpy(), g_cols.numpy())
        assert np.array_equal(want, pos.numpy())

    def mf_sgd_ordered(kind, P, Q, u, i, r, wu, wi, lr, reg_u, reg_i, loss, Bu=None, Bi=None, reg_b=0.0,
                       global_mean=0.0, n_warps=0):
        log.append(('mf_sgd_ordered', kind, n_warps))
        eu, ei = E.mf_order_prepare(u.numpy(), i.numpy(), P.shape[0], Q.shape[0])
        assert np.array_equal(eu, wu.numpy()) and np.array_equal(ei, wi.numpy())
        args = (P.numpy(), Q.numpy(), u.numpy(), i.numpy(), r.numpy(), lr, reg_u, reg_i)
        if kind in (1, 4):
            loss += float(SM.rating_pass(*args, copies=kind == 4))
        elif kind == 3:
            loss += float(_edge_pass(*args))
        else:
            assert kind == 5
            loss += float(EO.rating_pass(P.numpy(), Q.numpy(), Bu.numpy(), Bi.numpy(), *args[2:], reg_b, global_mean))

    def rste_sgd_ordered(P, Q, u, i, r, wu, wi, wr, pos_rowptr, pos, f_rowptr, f_cols, f_w, denom, lr, reg_u, reg_i,
                         alpha, loss, n_warps=0):
        log.append(('rste_sgd_ordered', None, n_warps))
        want = E.rste_order_prepare(u.numpy(), i.numpy(), P.shape[0], Q.shape[0], f_rowptr.numpy(), f_cols.numpy())
        assert all(np.array_equal(a, b.numpy()) for a, b in zip(want[:5], (wu, wi, wr, pos_rowptr, pos)))
        loss += float(_rste_pass(P.numpy(), Q.numpy(), u.numpy(), i.numpy(), r.numpy(), _lists(f_rowptr, f_cols, f_w),
                                 lr, reg_u, reg_i, alpha))

    def rste_predict_pairs(P, Q, u, i, f_rowptr, f_cols, f_w, denom, alpha, out=None):
        log.append(('rste_predict_pairs', None, None))
        fl = _lists(f_rowptr, f_cols, f_w)
        return torch.tensor([SR.rste_predict(P.numpy(), Q.numpy(), uu, ii, fl, alpha)
                             for uu, ii in zip(u.tolist(), i.tolist())], dtype=P.dtype)

    def social_user_pass(kind, P, visit, pos, f_rowptr, f_cols, f_val, g_rowptr, g_cols, g_val, lr, coef, loss,
                         n_warps=0):
        log.append(('social_user_pass', kind, n_warps))
        schedule_of(P, visit, pos, f_rowptr, f_cols, g_rowptr, g_cols)
        fl, v = _lists(f_rowptr, f_cols, f_val), visit.tolist()
        if kind == 0:
            loss += float(SM.socialmf_user_pass(P.numpy(), v, fl, lr, coef))
        else:
            loss += float(SM.soreg_user_pass(P.numpy(), v, fl, _lists(g_rowptr, g_cols, g_val), lr, coef))

    def sree_user_pass(P, visit, pos, f_rowptr, f_cols, f_w, g_rowptr, g_cols, lr, alpha, loss, n_warps=0):
        log.append(('sree_user_pass', None, n_warps))
        schedule_of(P, visit, pos, f_rowptr, f_cols, g_rowptr, g_cols)
        loss += float(EO.sree_user_pass(P.numpy(), visit.tolist(), _lists(f_rowptr, f_cols, f_w), lr, alpha))

    def sumsq(x, out):
        out += float((x.double() * x.double()).sum())

    def knn_pair_similarity(rowptr, cols, vals, sq, means, sorted_cols, sorted_vals, sorted_sq, a, b, w):
        log.append(('knn_pair_similarity', None, None))
        rows = [dict(zip(c.tolist(), v.tolist())) for c, v in _lists(rowptr, cols, vals)]
        return torch.tensor([(KO.similarity(rows[x], rows[y], 'pcc') + wk) / 2.0
                             for x, y, wk in zip(a.tolist(), b.tolist(), w.tolist())], dtype=torch.float64)

    monkeypatch.setattr(IterativeRecommender, '_device', lambda self: torch.device('cpu'))
    for f in (mf_sgd_ordered, rste_sgd_ordered, rste_predict_pairs, social_user_pass, sree_user_pass, sumsq,
              knn_pair_similarity):
        monkeypatch.setattr(E, f.__name__, f)
    return log


def _film(name):
    """A recorded FilmTrust run; the SREE file shares the lists of the EE one."""
    g = dict(np.load(os.path.join(GOLD, '%s_filmtrust.npz' % name.lower())))
    if name == 'SREE':
        ee = np.load(os.path.join(GOLD, 'ee_filmtrust.npz'))
        g.update({k: ee[k] for k in LISTS})
    return g


def _write_inputs(g, tmp_path):
    """The run's training, test and trust files (SoRec and RSTE recorded the cleaned relation list, the others the
    list as read) and its configuration pointing at them."""
    files = {'train.txt': ('train_users', 'train_items', 'train_rating'),
             'test.txt': ('test_users', 'test_items', 'test_rating')}
    if 'raw_u1' in g or 'rel_u1' in g:
        files['trust.txt'] = ('raw_u1', 'raw_u2', 'raw_w') if 'raw_u1' in g else ('rel_u1', 'rel_u2', 'rel_w')
    for fname, cols in files.items():
        (tmp_path / fname).write_text(''.join('%s %s %r\n' % x for x in zip(*(g[c].tolist() for c in cols))))
    return (str(g['conf']).replace('./dataset/FilmTrust/trainset.txt', 'train.txt')
            .replace('./dataset/FilmTrust/testset.txt', 'test.txt').replace('./dataset/FilmTrust/trust.txt', 'trust.txt'))


@pytest.mark.parametrize('name', ['SoRec', 'RSTE', 'SocialMF', 'SoReg', 'EE', 'SREE'])
def test_qrec_execute_reproduces_the_reference_filmtrust_run(name, calls, tmp_path, monkeypatch):
    from qrec_b200.QRec import QRec
    from qrec_b200.util.config import ModelConf
    g = _film(name)
    monkeypatch.chdir(tmp_path)
    (tmp_path / 'run.conf').write_text(_write_inputs(g, tmp_path))
    random.seed(int(g['seed']))
    np.random.seed(int(g['seed']))
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        measure = QRec(ModelConf('run.conf')).execute()
    lines = [ln for ln in out.getvalue().splitlines() if ' epoch ' in ln and 'loss = ' in ln]
    assert lines == g['epoch_lines'].tolist()
    assert [m.strip() for m in measure] == g['measure'].tolist()
    setup = [('knn_pair_similarity', None)] if name == 'SoReg' else []
    assert [c[:2] for c in calls] == setup + EPOCH[name] * len(lines)
    assert all(64 <= c[2] <= 2368 for c in calls if c[2] is not None)
