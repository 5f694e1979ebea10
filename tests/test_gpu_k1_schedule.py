"""The fused user-major BPR epoch against a float64 restatement of its wave semantics.

The epoch's launches run in waves (qrec_b200/csrc/um_waves.cuh).  Before a wave the item table is snapshotted; every
user of the wave runs its triples in order with P[u] updated after each one, reading item rows only from the snapshot;
the item-row deltas of the whole wave are summed into the table.  k1_wave_oracle.py does exactly that in float64, with
the negatives the GPU drew.  What is left between the two is fp32 rounding and the summation order of the
scatter-adds, far below the difference that one triple in a different wave would make."""
import numpy as np
import pytest

from k1_wave_oracle import CH, check_against, pipeline_launches, wave_chunks, wave_oracle  # noqa: F401

pytestmark = pytest.mark.gpu

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


def test_oracle_resolves_wave_membership(case):
    """Moving every wave boundary by one chunk moves about one user per wave into the neighbouring wave; the tables
    that gives must miss check_against's bound tenfold, or that bound would not pin the wave membership."""
    c = case
    Po, Qo, _ = c['oracle']
    Ps, Qs, _ = wave_oracle(c['P0'], c['Q0'], c['rowptr'], c['i'], c['j'], [(0, USERS)], LR, REG, shift=CH)
    for got, ref, init in ((Ps, Po, c['P0']), (Qs, Qo, c['Q0'])):
        assert np.abs(got - ref).max() > 1e-3 * np.abs(ref - init).max()


@pytest.mark.parametrize('entry', ['plain', 'sig'])
def test_fused_epoch_matches_wave_oracle(torch, E, case, entry):
    c = case
    dev = c['dev']
    P, Q = dev(c['P0']), dev(c['Q0'])
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    jo = torch.full((len(c['i']),), -1, dtype=torch.int32, device='cuda')
    args = (P, Q, dev(c['rowptr']), dev(c['i']), c['rrp'], c['rc'])
    if entry == 'plain':
        E.bpr_epoch_usermajor(*args, ITEMS, SEED, EPOCH, LR, REG, REG, loss, j_out=jo)
    else:
        E.bpr_epoch_usermajor_sig(*args, E.rated_signature(c['rrp'], c['rc']), ITEMS, SEED, EPOCH, LR, REG, REG, loss, j_out=jo)
    torch.cuda.synchronize()
    assert np.array_equal(jo.cpu().numpy(), c['j']), 'fused sampler != stand-alone Philox sampler'
    check_against(P.cpu().numpy(), Q.cpu().numpy(), loss.item(), c['P0'], c['Q0'], c['oracle'])


def test_host_pipeline_matches_wave_oracle(torch, E, case):
    """Small staging chunks: every chunk of whole users is a launch of its own, with waves sized for it."""
    c = case
    rowptr, chunk = c['rowptr'], 200_000
    launches = pipeline_launches(rowptr, chunk)
    assert len(launches) > 10
    oracle = wave_oracle(c['P0'], c['Q0'], rowptr, c['i'], c['j'], launches, LR, REG)
    P, Q = c['dev'](c['P0']), c['dev'](c['Q0'])
    pipe = E.HostPipeline(0, chunk_triples=chunk)
    hl = pipe.bpr_epoch_usermajor(P, Q, torch.from_numpy(rowptr).pin_memory(), torch.from_numpy(c['i']).pin_memory(),
                                  c['rrp'], c['rc'], ITEMS, SEED, EPOCH, LR, REG, REG)
    torch.cuda.synchronize()
    pipe.close()
    check_against(P.cpu().numpy(), Q.cpu().numpy(), hl, c['P0'], c['Q0'], oracle)
