"""The fused user-major BPR epoch against a float64 restatement of its wave semantics.

The epoch's launches run in waves (qrec_b200/csrc/um_waves.cuh).  Before a wave the item table is snapshotted; every
user of the wave runs its triples in order with P[u] updated after each one, reading item rows only from the snapshot;
the item-row deltas of the whole wave are summed into the table.  The oracle below does exactly that in float64, with
the negatives the GPU drew.  What is left between the two is fp32 rounding and the summation order of the
scatter-adds, far below the difference that one triple in a different wave would make."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CH = 32
LR, REG = 0.01, 0.001          # bench.py's learning rate and regularisation
USERS, ITEMS, D, MAXDEG = 50_000, 5_000, 64, 120
SEED, EPOCH = 0x5eed, 4


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def wave_chunks(n, num_items, d):
    """launch_usermajor's wave length in chunks of CH triples (um_wave_chunks)."""
    copy_bytes = 2 * num_items * d * 4
    copy_floor = 8 * copy_bytes // (24 * d + 12) if copy_bytes > (8 << 20) else 0
    return max(min(max(n // 64, copy_floor), 4 * num_items) // CH, 1)


def wave_oracle(P0, Q0, rowptr, i, j, launches, lr, reg, shift=0):
    """float64 epoch: launches = [(ua, ub)], each a separate launch over users [ua, ub) with its own waves.  shift
    moves every wave boundary `shift` triples earlier."""
    from scipy import sparse
    P, Q = P0.astype(np.float64), Q0.astype(np.float64)
    a = lr * reg
    loss = 0.0
    for ua, ub in launches:
        start = rowptr[ua:ub] - rowptr[ua]
        deg = np.diff(rowptr[ua:ub + 1])
        wave_of = (start + shift) // (wave_chunks(int(rowptr[ub] - rowptr[ua]), Q.shape[0], Q.shape[1]) * CH)
        users = np.arange(ua, ub)
        for w in np.unique(wave_of[deg > 0]):
            sel = (wave_of == w) & (deg > 0)
            uu, first, dg = users[sel], rowptr[ua:ub][sel], deg[sel]
            Qw = Q.copy()
            rows, deltas = [], []
            for k in range(int(dg.max())):
                on = dg > k
                u, t = uu[on], first[on] + k
                p, qi, qj = P[u], Qw[i[t]], Qw[j[t]]
                x = np.einsum('ij,ij->i', p, qi - qj)
                s = 1.0 / (1.0 + np.exp(-x))
                g = (lr * (1.0 - s))[:, None]
                loss += float(-np.log(s).sum())
                pn = p + g * (qi - qj)
                rows += [i[t], j[t]]
                deltas += [g * (1 - a) * pn - a * qi, -g * (1 - a) * pn - a * qj]
                P[u] = (1 - a) * pn
            r = np.concatenate(rows)
            S = sparse.csr_matrix((np.ones(len(r)), (r, np.arange(len(r)))), shape=(Q.shape[0], len(r)))
            Q += S @ np.concatenate(deltas)
    return P, Q, loss


@pytest.fixture(scope='module')
def case(torch, E):
    rng = np.random.default_rng(2024)
    deg = rng.integers(0, MAXDEG + 1, USERS)
    rowptr = np.zeros(USERS + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    u = np.repeat(np.arange(USERS), deg).astype(np.int32)
    i = np.concatenate([rng.choice(ITEMS, k, replace=False) for k in deg]).astype(np.int32)
    csr = E.RatedCSR(USERS, ITEMS, u, i)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
    rrp, rc = dev(csr.sorted_rowptr), dev(csr.sorted_cols)
    j = E.sample_neg_philox(dev(u), rrp, rc, ITEMS, SEED, EPOCH).cpu().numpy()
    P0 = (rng.random((USERS, D)) / 3).astype(np.float32)
    Q0 = (rng.random((ITEMS, D)) / 3).astype(np.float32)
    Po, Qo, lo = wave_oracle(P0, Q0, rowptr, i, j, [(0, USERS)], LR, REG)
    return dict(rowptr=rowptr, u=u, i=i, j=j, rrp=rrp, rc=rc, P0=P0, Q0=Q0, oracle=(Po, Qo, lo), dev=dev)


def check_against(got_P, got_Q, got_loss, P0, Q0, oracle):
    """fp32 tables and an fp32 loss per lane against float64: at this shape the rounding alone is about 3e-5 of the
    update on P.  Users run one wave early or late move the tables by far more (test_oracle_resolves_wave_membership)."""
    Po, Qo, lo = oracle
    errs = {}
    for got, ref, init, name in ((got_P, Po, P0, 'P'), (got_Q, Qo, Q0, 'Q')):
        update = np.abs(ref - init).max()
        err = np.abs(got.astype(np.float64) - ref).max()
        print('%s: max-abs error %.3g of an update of %.3g (ratio %.3g)' % (name, err, update, err / update))
        assert update > 0
        errs[name] = err / update
    print('loss: relative error %.3g' % (abs(got_loss - lo) / lo))
    assert errs['P'] <= 1e-4 and errs['Q'] <= 1e-4, errs
    assert abs(got_loss - lo) <= 1e-5 * lo


def test_oracle_resolves_wave_membership(case):
    """Moving every wave boundary by one chunk moves about one user per wave into the neighbouring wave; the tables
    that gives must miss check_against's bound tenfold, or that bound would not pin the wave membership."""
    c = case
    Po, Qo, _ = c['oracle']
    Ps, Qs, _ = wave_oracle(c['P0'], c['Q0'], c['rowptr'], c['i'], c['j'], [(0, USERS)], LR, REG, shift=CH)
    for got, ref, init in ((Ps, Po, c['P0']), (Qs, Qo, c['Q0'])):
        assert np.abs(got - ref).max() > 1e-3 * np.abs(ref - init).max()


@pytest.mark.parametrize('entry', ['plain', 'sig', 'tma'])
def test_fused_epoch_matches_wave_oracle(torch, E, case, entry):
    c = case
    dev = c['dev']
    P, Q = dev(c['P0']), dev(c['Q0'])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    jo = torch.full((len(c['i']),), -1, dtype=torch.int32, device='cuda')
    args = (P, Q, dev(c['rowptr']), dev(c['i']), c['rrp'], c['rc'])
    if entry == 'plain':
        E.bpr_epoch_usermajor(*args, ITEMS, SEED, EPOCH, LR, REG, REG, loss, j_out=jo)
    elif entry == 'sig':
        E.bpr_epoch_usermajor_sig(*args, E.rated_signature(c['rrp'], c['rc']), ITEMS, SEED, EPOCH, LR, REG, REG, loss, j_out=jo)
    else:
        E.bpr_epoch_usermajor_tma(*args, ITEMS, SEED, EPOCH, LR, REG, REG, loss, j_out=jo)
    torch.cuda.synchronize()
    assert np.array_equal(jo.cpu().numpy(), c['j']), 'fused sampler != stand-alone Philox sampler'
    check_against(P.cpu().numpy(), Q.cpu().numpy(), loss.item(), c['P0'], c['Q0'], c['oracle'])


def test_host_pipeline_matches_wave_oracle(torch, E, case):
    """Small staging chunks: every chunk of whole users is a launch of its own, with waves sized for it."""
    c = case
    rowptr, chunk = c['rowptr'], 200_000
    launches, ua = [], 0
    while ua < USERS:                                   # the pipeline's cut: the most whole users within `chunk` triples
        ub = int(np.searchsorted(rowptr, rowptr[ua] + chunk, side='right')) - 1
        ub = min(max(ub, ua + 1), USERS, ua + chunk)
        launches.append((ua, ub))
        ua = ub
    assert len(launches) > 10
    oracle = wave_oracle(c['P0'], c['Q0'], rowptr, c['i'], c['j'], launches, LR, REG)
    P, Q = c['dev'](c['P0']), c['dev'](c['Q0'])
    pipe = E.HostPipeline(0, chunk_triples=chunk)
    hl = pipe.bpr_epoch_usermajor(P, Q, torch.from_numpy(rowptr).pin_memory(), torch.from_numpy(c['i']).pin_memory(),
                                  c['rrp'], c['rc'], ITEMS, SEED, EPOCH, LR, REG, REG)
    torch.cuda.synchronize()
    pipe.close()
    check_against(P.cpu().numpy(), Q.cpu().numpy(), hl, c['P0'], c['Q0'], oracle)
