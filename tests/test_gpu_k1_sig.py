"""The signature pre-test in the fused sampler (qrec_bpr_epoch_usermajor_sig_f32): the 512-bit rated-set
signature has no false negatives, so the sampled negatives must be bit-identical to the plain fused
kernel and to the stand-alone Philox sampler.  Needs a GPU."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

REG = 0.001


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _signature(rowptr, cols):
    sig = np.zeros((len(rowptr) - 1, 16), np.uint32)
    for u in range(len(rowptr) - 1):
        for c in cols[rowptr[u]:rowptr[u + 1]].tolist():
            sig[u, (c >> 5) & 15] |= np.uint32(1) << np.uint32(c & 31)
    return sig


def _problem(E, nu, ni, rng, heavy=None):
    deg = rng.integers(0, 60, nu)
    deg[3] = 0
    if heavy:
        deg[7] = heavy                                      # saturates the signature: always bisects
    u = np.repeat(np.arange(nu), deg)
    i = np.concatenate([rng.choice(ni, k, replace=False) for k in deg]).astype(np.int32) if len(u) else np.zeros(0, np.int32)
    return E.RatedCSR(nu, ni, u, i)


def test_signature_build_matches_numpy(torch, E):
    rng = np.random.default_rng(0)
    csr = _problem(E, 500, 3000, rng, heavy=1500)
    sig = E.rated_signature(_dev(torch, csr.sorted_rowptr), _dev(torch, csr.sorted_cols))
    torch.cuda.synchronize()
    got = sig.cpu().numpy().view(np.uint32)
    assert np.array_equal(got, _signature(csr.sorted_rowptr, csr.sorted_cols))
    # user 3 has no rated items; the heavy user's 1500 items set (nearly) every one of the 512 bits
    assert not got[3].any() and sum(bin(int(w)).count('1') for w in got[7]) >= 0.9 * 512


@pytest.mark.parametrize('d', [16, 32, 64, 128])
def test_sig_epoch_draws_the_same_negatives_and_applies_the_same_updates(torch, E, d):
    rng = np.random.default_rng(d)
    nu, ni = 3000, 700                                       # small item set: ~5 % of the draws are rejected
    csr = _problem(E, nu, ni, rng, heavy=600)
    cu = np.repeat(np.arange(nu), np.diff(csr.pos_rowptr)).astype(np.int32)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32); Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    Pa, Qa, Pb, Qb = _dev(torch, P0), _dev(torch, Q0), _dev(torch, P0), _dev(torch, Q0)
    rp, ci = _dev(torch, csr.pos_rowptr), _dev(torch, csr.pos_cols)
    rrp, rc = _dev(torch, csr.sorted_rowptr), _dev(torch, csr.sorted_cols)
    sig = E.rated_signature(rrp, rc)
    la = torch.zeros(1, dtype=torch.float64, device='cuda'); lb = torch.zeros(1, dtype=torch.float64, device='cuda')
    ja = torch.full((len(cu),), -1, dtype=torch.int32, device='cuda'); jb = ja.clone()
    lr = 1e-4
    E.bpr_epoch_usermajor(Pa, Qa, rp, ci, rrp, rc, ni, 0xabcdef, 3, lr, REG, REG, la, j_out=ja)
    E.bpr_epoch_usermajor_sig(Pb, Qb, rp, ci, rrp, rc, sig, ni, 0xabcdef, 3, lr, REG, REG, lb, j_out=jb)
    torch.cuda.synchronize()
    assert torch.equal(ja, jb)
    assert torch.equal(jb, E.sample_neg_philox(_dev(torch, cu), rrp, rc, ni, 0xabcdef, 3))
    # no negative is a rated item
    rated = set(zip(np.repeat(np.arange(nu), np.diff(csr.sorted_rowptr)).tolist(), csr.sorted_cols.tolist()))
    assert not any((a, b) in rated for a, b in zip(cu.tolist(), jb.cpu().numpy().tolist()))
    P0t, Q0t = _dev(torch, P0), _dev(torch, Q0)
    dPa, dPb, dQa, dQb = Pa - P0t, Pb - P0t, Qa - Q0t, Qb - Q0t
    assert float((dPa - dPb).abs().max()) <= 0.02 * float(dPa.abs().max())
    assert float((dQa - dQb).abs().max()) <= 0.02 * float(dQa.abs().max())
    assert abs(la.item() - lb.item()) <= 1e-4 * abs(la.item())


def test_sig_entry_point_rejects_bad_arguments(torch, E):
    P = torch.zeros(4, 20, device='cuda'); Q = torch.zeros(5, 20, device='cuda')
    rp = torch.zeros(5, dtype=torch.int64, device='cuda'); ci = torch.zeros(0, dtype=torch.int32, device='cuda')
    sig = torch.zeros(4, 16, dtype=torch.int32, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    with pytest.raises(E.QRecError):                         # d = 20: not a full-lane configuration
        E.bpr_epoch_usermajor_sig(P, Q, rp, ci, rp, ci, sig, 5, 1, 0, 0.1, 0.0, 0.0, loss)
    with pytest.raises(E.QRecError):                         # signature of the wrong shape
        E.bpr_epoch_usermajor_sig(P, Q, rp, ci, rp, ci, sig[:2], 5, 1, 0, 0.1, 0.0, 0.0, loss)
