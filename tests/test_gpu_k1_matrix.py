"""Every instantiation of the user-major BPR epoch against the float64 wave oracle (k1_wave_oracle.py).

bpr_sgd_usermajor_kernel<LPR, G, FULL, SAMPLE, MINB, SIG> (bpr_kernels.cu) is compiled for four lane-group sizes, each
with and without idle lanes, with the negatives given or drawn in the kernel (plain, signature pre-test), and
launch_usermajor sizes its waves by three rules.  The cases of k1_wave_oracle.CASES reach all of them
(test_k1_wave_oracle_cpu.py proves that without a GPU): ragged degrees around the lane-group size and the number of
triples in flight, users longer than a wave whose items repeat, a saturated user, the 4 x items cap and the snapshot-copy
floor of the wave length, a launch with fewer triples than users, and the host pipeline's chunked launches.  The
regularisers differ, the rejection sets are a strict superset of the positives, and the Philox key uses the high half
of the seed and the top bit of the epoch.

Each case's bound is at most 3 x the error observed on an H100 80GB HBM3 (700 W power limit) and at least 10 x under
what the oracle with every wave boundary moved by one chunk gives, so it pins the wave a user runs in."""
import functools

import numpy as np
import pytest

from k1_wave_oracle import CASES, CH, case_data, case_launches, case_tables, check_against, table_ratios, wave_oracle

pytestmark = pytest.mark.gpu

LR, REG_U, REG_I = 0.01, 0.001, 0.003


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@functools.lru_cache(maxsize=1)                  # the entries of one case run back to back
def prepared(case):
    """The case's triples, the stand-alone sampler's negatives, the oracle, and how far the oracle with every wave
    boundary one chunk early lies from it."""
    from qrec_b200 import engine as E
    c = case_data(case, E)
    c['rrp'], c['rc'] = dev(c['rated_rowptr']), dev(c['rated_cols'])
    c['j'] = E.sample_neg_philox(dev(c['u']), c['rrp'], c['rc'], case.items, *case.key).cpu().numpy()
    c['P0'], c['Q0'] = case_tables(case)
    launches = case_launches(case, c['rowptr'])
    c['oracle'] = wave_oracle(c['P0'], c['Q0'], c['rowptr'], c['i'], c['j'], launches, LR, REG_U, REG_I)
    shifted = wave_oracle(c['P0'], c['Q0'], c['rowptr'], c['i'], c['j'], launches, LR, REG_U, REG_I, shift=CH)
    c['shifted'] = table_ratios(shifted[0], shifted[1], c['P0'], c['Q0'], c['oracle'])
    return c


def test_negatives_respect_the_rejection_sets(torch, E):
    """What the cases are built to draw: no negative is a rated item, sub-threshold ones included, except for the
    saturated user, who takes first draws; and the long users' draws are mostly rejected at least once."""
    from k1_wave_oracle import LONG_USERS, SATURATED_USER
    case = next(c for c in CASES if c.name == 'long64')
    c = prepared(case)
    rated = np.zeros((case.users, case.items), bool)
    rated[np.repeat(np.arange(case.users), np.diff(c['rated_rowptr'])), c['rated_cols']] = True
    hit = rated[c['u'], c['j']]
    assert hit[c['u'] == SATURATED_USER].all() and not hit[c['u'] != SATURATED_USER].any()
    assert (c['j'] == c['i'])[c['u'] == SATURATED_USER].any()
    first = E.sample_neg_philox(dev(c['u']), dev(np.zeros(case.users + 1, np.int64)), c['rc'], case.items,
                                *case.key).cpu().numpy()           # empty rejection sets: every first draw
    long_user = np.isin(c['u'], list(LONG_USERS))
    assert (first != c['j'])[long_user].mean() > 0.5


@pytest.mark.parametrize('case,entry', [(c, e) for c in CASES for e in c.entries],
                         ids=['%s-%s' % (c.name, e) for c in CASES for e in c.entries])
def test_epoch_matches_wave_oracle(torch, E, case, entry):
    c = prepared(case)
    seed, epoch = case.key
    P, Q = dev(c['P0']), dev(c['Q0'])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    jo = torch.full((len(c['i']),), -1, dtype=torch.int32, device='cuda') if entry in ('plain', 'sig') else None
    if entry in ('pipe', 'pipe_sig'):
        pipe = E.HostPipeline(0, chunk_triples=case.chunk)
        if entry == 'pipe_sig':
            # taken by the kernel only where every lane owns a slice (d = 16, 32, 64, 128); elsewhere the plain sampler runs
            pipe.set_rated_signature(E.rated_signature(c['rrp'], c['rc']))
        got_loss = pipe.bpr_epoch_usermajor(P, Q, torch.from_numpy(c['rowptr']).pin_memory(),
                                            torch.from_numpy(c['i']).pin_memory(), c['rrp'], c['rc'], case.items, seed, epoch,
                                            LR, REG_U, REG_I)
        torch.cuda.synchronize()
        pipe.close()
    else:
        args = (P, Q, dev(c['rowptr']), dev(c['i']), c['rrp'], c['rc'])
        if entry == 'given':
            E.bpr_sgd_usermajor(P, Q, dev(c['rowptr']), dev(c['i']), dev(c['j']), LR, REG_U, REG_I, loss)
        elif entry == 'sig':
            E.bpr_epoch_usermajor_sig(*args, E.rated_signature(c['rrp'], c['rc']), case.items, seed, epoch, LR, REG_U, REG_I,
                                      loss, j_out=jo)
        else:
            E.bpr_epoch_usermajor(*args, case.items, seed, epoch, LR, REG_U, REG_I, loss, j_out=jo)
        torch.cuda.synchronize()
        got_loss = loss.item()
    if jo is not None:
        assert np.array_equal(jo.cpu().numpy(), c['j']), 'fused sampler != stand-alone Philox sampler'
    print('\n%s-%s: boundaries one chunk early move P by %.3g and Q by %.3g of the largest update'
          % (case.name, entry, c['shifted']['P'], c['shifted']['Q']))
    check_against(P.cpu().numpy(), Q.cpu().numpy(), got_loss, c['P0'], c['Q0'], c['oracle'], case.tol, case.loss_tol)
    assert c['shifted']['P'] >= 10 * case.tol[0] and c['shifted']['Q'] >= 10 * case.tol[1], \
        'the bound cannot tell a user in the wrong wave'
