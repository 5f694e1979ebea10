"""The waves of one user-major epoch call are chained with programmatic dependent launch (bpr_kernels.cu:
launch_usermajor): each wave's snapshot copy (um_snapshot_kernel) and K1 may start before their predecessor on the
stream ends, and K1 reads its users' P rows, i and negatives before it waits.  These tests pin what that must not
change: the copy is exact, the first wave still sees every earlier write on the stream, consecutive calls compose, and
the negatives stay those of the stand-alone sampler."""
import numpy as np
import pytest

from test_gpu_k1_schedule import CH, EPOCH, ITEMS, LR, REG, SEED, check_against, wave_oracle  # noqa: F401

pytestmark = pytest.mark.gpu

USERS, D, MAXDEG = 20_000, 64, 120


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


@pytest.mark.parametrize('rows', [1, 3, 100_000, 1_000_003])
def test_snapshot_copy_is_bit_exact(torch, E, rows):
    """Tiny tables (less than one float4 per thread), the benchmark's 100K x 64 item table and a 1M-row one."""
    src = torch.randn(rows, D, device='cuda')
    src.view(-1)[::7] = float('nan')          # every bit pattern survives, NaNs included
    dst = torch.full_like(src, 3.0)
    E.table_snapshot(src, dst)
    torch.cuda.synchronize()
    assert torch.equal(src.view(torch.int32), dst.view(torch.int32))


@pytest.fixture(scope='module')
def case(torch, E):
    rng = np.random.default_rng(77)
    deg = rng.integers(0, MAXDEG + 1, USERS)
    rowptr = np.zeros(USERS + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    u = np.repeat(np.arange(USERS), deg).astype(np.int32)
    i = np.concatenate([rng.choice(ITEMS, k, replace=False) for k in deg]).astype(np.int32)
    csr = E.RatedCSR(USERS, ITEMS, u, i)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
    rrp, rc = dev(csr.sorted_rowptr), dev(csr.sorted_cols)
    P0 = (rng.random((USERS, D)) / 3).astype(np.float32)
    Q0 = (rng.random((ITEMS, D)) / 3).astype(np.float32)
    return dict(rowptr=rowptr, u=u, i=i, rrp=rrp, rc=rc, sig=E.rated_signature(rrp, rc), P0=P0, Q0=Q0, dev=dev)


def negatives(torch, E, c, epoch):
    return E.sample_neg_philox(c['dev'](c['u']), c['rrp'], c['rc'], ITEMS, SEED, epoch).cpu().numpy()


def epoch_call(torch, E, c, P, Q, epoch, loss, jo):
    E.bpr_epoch_usermajor_sig(P, Q, c['dev'](c['rowptr']), c['dev'](c['i']), c['rrp'], c['rc'], c['sig'], ITEMS, SEED, epoch,
                              LR, REG, REG, loss, j_out=jo)


def test_first_wave_sees_a_kernel_run_just_before_it(torch, E, case):
    """P and Q are rewritten by kernels queued on the same stream right before the epoch, with no synchronisation in
    between: the epoch must start from the rewritten tables, so wave 0's early prologue (its P rows) and its snapshot
    both respect stream order."""
    c = case
    P, Q = c['dev'](np.zeros_like(c['P0'])), c['dev'](np.zeros_like(c['Q0']))
    torch.cuda.synchronize()
    P_src, Q_src = c['dev'](c['P0']), c['dev'](c['Q0'])
    torch.cuda.synchronize()
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    jo = torch.full((len(c['i']),), -1, dtype=torch.int32, device='cuda')
    torch.cuda._sleep(50_000_000)             # keeps the stream busy so the epoch is queued behind the rewrites
    P.copy_(P_src)
    Q.copy_(Q_src)
    P.mul_(0.5)
    Q.mul_(1.5)
    epoch_call(torch, E, c, P, Q, EPOCH, loss, jo)
    torch.cuda.synchronize()
    j = negatives(torch, E, c, EPOCH)
    assert np.array_equal(jo.cpu().numpy(), j), 'fused sampler != stand-alone Philox sampler'
    P1, Q1 = c['P0'] * np.float32(0.5), c['Q0'] * np.float32(1.5)
    oracle = wave_oracle(P1, Q1, c['rowptr'], c['i'], j, [(0, USERS)], LR, REG)
    check_against(P.cpu().numpy(), Q.cpu().numpy(), loss.item(), P1, Q1, oracle)


def test_two_back_to_back_epochs_match_the_oracle_applied_twice(torch, E, case):
    c = case
    P, Q = c['dev'](c['P0']), c['dev'](c['Q0'])
    losses = torch.zeros(2, dtype=torch.float64, device='cuda')
    jo = [torch.full((len(c['i']),), -1, dtype=torch.int32, device='cuda') for _ in range(2)]
    for k in range(2):
        epoch_call(torch, E, c, P, Q, EPOCH + k, losses[k:k + 1], jo[k])
    torch.cuda.synchronize()
    Po, Qo = c['P0'], c['Q0']
    for k in range(2):
        j = negatives(torch, E, c, EPOCH + k)
        assert np.array_equal(jo[k].cpu().numpy(), j), 'fused sampler != stand-alone Philox sampler (epoch %d)' % k
        Pn, Qn, ln = wave_oracle(Po, Qo, c['rowptr'], c['i'], j, [(0, USERS)], LR, REG)
        if k == 0:
            P_first, Q_first, l_first = Pn, Qn, ln
        Po, Qo = Pn, Qn
    check_against(P.cpu().numpy(), Q.cpu().numpy(), losses[1].item(), c['P0'], c['Q0'], (Po, Qo, ln))
    assert abs(losses[0].item() - l_first) <= 1e-5 * l_first
