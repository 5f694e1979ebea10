"""Every lane-group instantiation of the row-parallel kernels outside the user-major BPR epoch against float64
references (row_shape_cases.py): the SpMM family, K3 in its four entries, the staged BPR step, the MF batch step in
its three kinds, the MF ordered step in float32 and float64 and the SVD++ user-major epoch.

Each launcher runs over its width table, which reaches every (LPR, VPL) or E it is compiled for with all lanes busy
and with idle lanes, and over row structures built to reach its masks and tails (test_row_shape_cases_cpu.py proves
both without a GPU).  Every case has an exact contract: conflict-free batches, distinct rows, one SVD++ user in flight
or users with disjoint items, so the reference is the kernel's own semantics and what is left is rounding.  Outputs
that the launch must not touch (rows no entry names, padding columns) are compared bit for bit.

Each bound is about 3 x the error observed on an H100 80GB HBM3 at 700 W (row_shape_cases.BOUNDS), and each test
rebuilds its reference with a plausible defect -- the last entry of every row dropped, the last float4 slice of a
lane group left out, or, for the parity kernel, the last element left out -- and asserts that it lies at least 10
bounds away."""
import numpy as np
import pytest

import row_shape_cases as R

pytestmark = pytest.mark.gpu

LR, REG_U, REG_I, REG_B, GLOBAL_MEAN = 0.01, 0.01, 0.02, 0.03, 3.0
SVDPP_REGS = (0.01, 0.01, 0.1, 0.01)                  # reg_u, reg_i, reg_b, reg_y
ACC_SCALE = -0.75


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def dev(x, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return t if dtype is None else t.to(dtype)


def host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def untouched(got, init, rows):
    """Rows outside `rows` keep their bits."""
    keep = np.ones(len(init), bool)
    keep[np.asarray(rows, np.int64)] = False
    assert R.same_bits(got[keep], init[keep]), 'rows the launch does not name were written'


def with_last_slice_of(bad, init, d):
    bad = np.array(bad, copy=True)
    bad[:, d - 4:] = init[:, d - 4:]
    return bad


# ------------------------------------------------------------------------------------------------------- SpMM
SPMM = ('spmm_balanced', 'spmm_rowsplit', 'spmm_scatter_rows', 'spmm_rows')


@pytest.mark.parametrize('launcher,d,structure', [(k, d, s) for k in SPMM for d in R.widths(k) for s in ('tails', 'long')],
                         ids=['%s-d%d-%s' % (k, d, s) for k in SPMM for d in R.widths(k) for s in ('tails', 'long')])
def test_spmm(torch, E, launcher, d, structure):
    c = R.spmm_case(launcher, d, structure)
    ref, terms = R.spmm_reference(launcher, c)
    bad, _ = R.spmm_reference(launcher, c, drop_last=True)
    csr = dev(c['rowptr']), dev(c['cols']), dev(c['vals'])
    X, acc = dev(c['X']), dev(c['acc0'])
    acc0 = c['acc0'].astype(np.float64)
    if launcher == 'spmm_rows':
        listed = c['rows'][c['rows'] >= 0]
        Y0 = np.full((c['n_rows'], d), 7.0, np.float32)
        Y = dev(Y0)
        E.spmm_csr_rows(*csr, dev(c['rows']), X, Y, acc=acc, acc_scale=ACC_SCALE)
        got_Y, got_acc = host(Y), host(acc)
        untouched(got_Y, Y0, listed)
        untouched(got_acc, c['acc0'], listed)
        got_Y, got_acc, acc0 = got_Y[listed], got_acc[listed], acc0[listed]
    else:
        Y = torch.full((c['n_cols'] if launcher == 'spmm_scatter_rows' else c['n_rows'], d), 3.0, device='cuda')
        if launcher == 'spmm_scatter_rows':
            E.spmm_csr_scatter_rows(*csr, dev(c['rows']), X, Y, acc=acc, acc_scale=ACC_SCALE)
        else:
            E.spmm_csr(*csr, X, Y, acc=acc, acc_scale=ACC_SCALE, rowsplit=launcher == 'spmm_rowsplit')
        got_Y, got_acc = host(Y), host(acc)
    acc_terms = np.abs(acc0) + abs(ACC_SCALE) * terms
    R.judge('%s d=%d %s' % (launcher, d, structure), R.BOUNDS[launcher], {
        'Y': (R.sum_ratio(got_Y, ref, terms), R.sum_ratio(bad, ref, terms)),
        'acc': (R.sum_ratio(got_acc, acc0 + ACC_SCALE * ref, acc_terms),
                R.sum_ratio(acc0 + ACC_SCALE * bad, acc0 + ACC_SCALE * ref, acc_terms)),
    })


# ------------------------------------------------------------------------------------------------------- K3
K3_EPS, K3_REG, LOG_WEIGHT = 1e-7, 0.01, 0.75


@pytest.mark.parametrize('entry', R.K3_ENTRIES)
@pytest.mark.parametrize('structure', list(R.K3_SIZES))
@pytest.mark.parametrize('d', R.widths('k3'))
def test_k3(torch, E, d, structure, entry):
    c = R.k3_case(d, structure)
    U, V, u, i, j = c['U'], c['V'], c['u'], c['i'], c['j']
    extra = dict(y_scale=c['y_scale'], y_full=c['y_full'], log_weight=LOG_WEIGHT)
    ref_loss, ref_gU, ref_gV, ref_y = R.k3_reference(U, V, u, i, j, K3_EPS, K3_REG, entry, **extra)
    bad_tabs = R.zero_last_slice([U, V], d)
    _, bad_gU, bad_gV, bad_y = R.k3_reference(*bad_tabs, u, i, j, K3_EPS, K3_REG, entry, **extra)
    last = np.nonzero(u >= 0)[0][-1]                # the loss defect: the batch's last triple left out
    u_short = u.copy()
    u_short[last] = -1
    bad_loss = R.k3_reference(U, V, u_short, i, j, K3_EPS, K3_REG, entry, **extra)[0]
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    args = dev(U), dev(V), dev(u), dev(i), dev(j)
    name = 'k3 %s d=%d %s' % (entry, d, structure)
    if entry == 'partial_scores':
        y = torch.full((len(u),), 7.0, device='cuda')
        E.bpr_partial_scores(*args, K3_REG, y, loss)
        ok = u >= 0
        pu = np.abs(U[u[ok]].astype(np.float64))
        terms = np.zeros(len(u))                    # skipped triples have no terms: their score must be exactly 0
        terms[ok] = (pu * np.abs(V[i[ok]]) + pu * np.abs(V[j[ok]])).sum(1)
        R.judge(name, R.BOUNDS['k3'], {
            'y': (R.sum_ratio(host(y), ref_y, terms), R.sum_ratio(bad_y, ref_y, terms)),
            'loss': (R.loss_ratio(loss.item(), ref_loss), R.loss_ratio(bad_loss, ref_loss)),
        })
        return
    gU, gV = dev(c['gU0']), dev(c['gV0'])
    if entry == 'grad':
        E.bpr_grad_scatter(*args, K3_EPS, K3_REG, gU, gV, loss)
    elif entry == 'scaled':
        E.bpr_grad_scatter_scaled(*args, dev(c['y_scale']), K3_EPS, K3_REG, gU, gV, loss)
    else:
        E.bpr_grad_from_scores(*args, dev(c['y_full']), K3_EPS, K3_REG, LOG_WEIGHT, gU, gV, loss)
    got_gU, got_gV = host(gU), host(gV)
    ok = u >= 0
    untouched(got_gU, c['gU0'], u[ok])
    untouched(got_gV, c['gV0'], np.concatenate([i[ok], j[ok]]))
    gU0, gV0 = c['gU0'].astype(np.float64), c['gV0'].astype(np.float64)
    R.judge(name, R.BOUNDS['k3'], {
        'gU': (R.table_ratio(got_gU, gU0 + ref_gU), R.table_ratio(gU0 + bad_gU, gU0 + ref_gU)),
        'gV': (R.table_ratio(got_gV, gV0 + ref_gV), R.table_ratio(gV0 + bad_gV, gV0 + ref_gV)),
        'loss': (R.loss_ratio(loss.item(), ref_loss), R.loss_ratio(bad_loss, ref_loss)),
    })


# ------------------------------------------------------------------------------------------------------- staged BPR
@pytest.mark.parametrize('structure', ['ragged', 'grid_stride'])
@pytest.mark.parametrize('d', R.widths('bpr_staged'))
def test_bpr_staged(torch, E, d, structure):
    c = R.staged_case(d, structure)
    u, pi, pj = c['u'], c['pos_i'], c['pos_j']
    ref_P, ref_D, ref_loss = R.staged_reference(c['P'], c['R'], c['D0'], u, pi, pj, LR, REG_U, REG_I)
    Pz, Rz = R.zero_last_slice([c['P'], c['R']], d)
    bad_P, bad_D, bad_loss = R.staged_reference(Pz, Rz, c['D0'], u, pi, pj, LR, REG_U, REG_I)
    bad_P, bad_D = with_last_slice_of(bad_P, c['P'], d), with_last_slice_of(bad_D, c['D0'], d)
    P, D = dev(c['P']), dev(c['D0'])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_staged(P, dev(u), dev(pi), dev(pj), dev(c['R']), D, LR, REG_U, REG_I, loss)
    got_P, got_D = host(P), host(D)
    untouched(got_P, c['P'], u)
    untouched(got_D, c['D0'], np.concatenate([pi, pj]))
    # the rows of D the launch writes, in units of the staged rows' rounding
    w, rows = np.concatenate([pi, pj]), np.abs(c['R']).max()
    R.judge('bpr_staged d=%d %s (%d triples)' % (d, structure, len(u)), R.BOUNDS['bpr_staged'], {
        'P': (R.table_ratio(got_P, ref_P), R.table_ratio(bad_P, ref_P)),
        'D': (R.table_ratio(got_D[w], ref_D[w], scale=rows), R.table_ratio(bad_D[w], ref_D[w], scale=rows)),
        'loss': (R.loss_ratio(loss.item(), ref_loss), R.loss_ratio(bad_loss, ref_loss)),
    })


# ------------------------------------------------------------------------------------------------------- MF
@pytest.mark.parametrize('kind', [0, 1, 2], ids=['BasicMF', 'PMF', 'SVD'])
@pytest.mark.parametrize('structure', ['ragged', 'windowed'])
@pytest.mark.parametrize('d', R.widths('mf_batch'))
def test_mf_batch(torch, E, d, structure, kind):
    from oracle import mf_oracle as M
    c = R.mf_batch_case(d, structure)
    u, i, r = c['u'], c['i'], c['r']
    regs = (LR, REG_U, REG_I)

    def reference(P, Q):
        dP, dQ, dBu, dBi, l = M.mf_sgd_jacobi(kind, P, Q, u, i, r, *regs, c['Bu'], c['Bi'], REG_B, GLOBAL_MEAN)
        return P + dP, Q + dQ, c['Bu'] + dBu, c['Bi'] + dBi, l
    ref = reference(c['P'].astype(np.float64), c['Q'].astype(np.float64))
    Pz, Qz = R.zero_last_slice([c['P'], c['Q']], d)
    bad = list(reference(Pz.astype(np.float64), Qz.astype(np.float64)))
    bad[0], bad[1] = with_last_slice_of(bad[0], c['P'], d), with_last_slice_of(bad[1], c['Q'], d)
    P, Q, Bu, Bi = dev(c['P']), dev(c['Q']), dev(c['Bu']), dev(c['Bi'])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.mf_sgd_batch(kind, P, Q, dev(u), dev(i), dev(r), *regs, loss, Bu if kind == 2 else None, Bi if kind == 2 else None,
                   REG_B, GLOBAL_MEAN, max_inflight=c['max_inflight'])
    got = [host(t) for t in (P, Q, Bu, Bi)]
    for t in got[:2]:
        assert not t[:, d - R.PAD:].any(), 'a padding column moved'
    untouched(got[0], c['P'], u)
    untouched(got[1], c['Q'], i)
    outputs = {'P': (R.table_ratio(got[0], ref[0]), R.table_ratio(bad[0], ref[0])),
               'Q': (R.table_ratio(got[1], ref[1]), R.table_ratio(bad[1], ref[1]))}
    if kind == 2:
        untouched(got[2], c['Bu'], u)
        untouched(got[3], c['Bi'], i)
        outputs['Bu'] = (R.table_ratio(got[2], ref[2]), R.table_ratio(bad[2], ref[2]))
        outputs['Bi'] = (R.table_ratio(got[3], ref[3]), R.table_ratio(bad[3], ref[3]))
    else:
        assert R.same_bits(got[2], c['Bu']) and R.same_bits(got[3], c['Bi'])
    outputs['loss'] = (R.loss_ratio(loss.item(), ref[4]), R.loss_ratio(bad[4], ref[4]))
    R.judge('mf_batch kind=%d d=%d %s' % (kind, d, structure), R.BOUNDS['mf_batch'], outputs)


@pytest.mark.parametrize('kind', [0, 1, 2], ids=['BasicMF', 'PMF', 'SVD'])
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('d', R.widths('mf_ordered'))
def test_mf_ordered(torch, E, d, dtype, kind):
    from oracle import c_oracle
    dt = np.dtype(dtype).type
    c = R.mf_ordered_case(d, dt)
    u, i, r = c['u'], c['i'], c['r']
    nu, ni = len(c['P']), len(c['Q'])

    def reference(cols):
        """float64 sequential pass over the columns [0, cols); the others keep their values."""
        P, Q = c['P'].astype(np.float64), c['Q'].astype(np.float64)
        Bu, Bi = c['Bu'].astype(np.float64), c['Bi'].astype(np.float64)
        Pc, Qc = np.ascontiguousarray(P[:, :cols]), np.ascontiguousarray(Q[:, :cols])
        l = c_oracle.mf_sgd_sequential(kind, Pc, Qc, u, i, r.astype(np.float64), LR, REG_U, REG_I,
                                       Bu if kind == 2 else None, Bi if kind == 2 else None, REG_B, GLOBAL_MEAN)
        P[:, :cols], Q[:, :cols] = Pc, Qc
        return P, Q, Bu, Bi, l
    ref, bad = reference(d), reference(d - 1)
    P, Q, Bu, Bi = dev(c['P']), dev(c['Q']), dev(c['Bu']), dev(c['Bi'])
    wu, wi = E.mf_order_prepare(u, i, nu, ni)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.mf_sgd_ordered(kind, P, Q, dev(u), dev(i), dev(r), dev(wu), dev(wi), LR, REG_U, REG_I, loss,
                     Bu if kind == 2 else None, Bi if kind == 2 else None, REG_B, GLOBAL_MEAN)
    got = [host(t) for t in (P, Q, Bu, Bi)]
    unit = R.U32 if dtype == 'float32' else R.U64
    names = ('P', 'Q', 'Bu', 'Bi') if kind == 2 else ('P', 'Q')
    outputs = {k: (R.table_ratio(got[n], ref[n], unit), R.table_ratio(bad[n], ref[n], unit)) for n, k in enumerate(names)}
    if kind != 2:
        assert R.same_bits(got[2], c['Bu']) and R.same_bits(got[3], c['Bi'])
    outputs['loss'] = (R.loss_ratio(loss.item(), ref[4], unit), R.loss_ratio(bad[4], ref[4], unit))
    R.judge('mf_ordered %s kind=%d d=%d' % (dtype, kind, d), R.BOUNDS['mf_ordered_' + ('f32' if dtype == 'float32' else 'f64')],
            outputs)


# ------------------------------------------------------------------------------------------------------- SVD++
@pytest.mark.parametrize('structure', ['one_in_flight', 'disjoint'])
@pytest.mark.parametrize('d', R.widths('svdpp_usermajor'))
def test_svdpp_usermajor(torch, E, d, structure):
    from oracle import svdpp_oracle as S
    c = R.svdpp_case(d, structure)
    csr = c['rowptr'], c['cols'], c['vals']

    def reference(tabs):
        ref = [t.astype(np.float64) for t in tabs]
        l = S.svdpp_usermajor(*ref, *csr, c['order'], LR, *SVDPP_REGS, GLOBAL_MEAN)
        return ref, l
    ref, ref_loss = reference(c['tabs'])
    bad, bad_loss = reference(R.zero_last_slice(c['tabs'], d))
    bad = [with_last_slice_of(b, t, d) if t.ndim == 2 else b for b, t in zip(bad, c['tabs'])]
    tabs = [dev(t) for t in c['tabs']]
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.svdpp_epoch_usermajor(*tabs, dev(c['rowptr']), dev(c['cols']), dev(c['vals']), dev(c['order']), LR, *SVDPP_REGS,
                            GLOBAL_MEAN, loss, max_users_in_flight=c['in_flight'])
    got = [host(t) for t in tabs]
    for t in got[:3]:
        assert not t[:, d - R.PAD:].any(), 'a padding column moved'
    users = np.nonzero(np.diff(c['rowptr']))[0]
    for t, init, rows in zip(got, c['tabs'], (users, c['cols'], c['cols'], users, c['cols'])):
        untouched(t, init, rows)
    outputs = {k: (R.table_ratio(g, x), R.table_ratio(b, x)) for k, g, x, b in zip(('P', 'Q', 'Y', 'Bu', 'Bi'), got, ref, bad)}
    outputs['loss'] = (R.loss_ratio(loss.item(), ref_loss), R.loss_ratio(bad_loss, ref_loss))
    R.judge('svdpp_usermajor d=%d %s' % (d, structure), R.BOUNDS['svdpp_usermajor'], outputs)
