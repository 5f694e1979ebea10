"""Edge cases of the C ABI on the device: empty inputs are no-ops, bad arguments come back as error
codes with a message (never a crash), and maximum supported widths run."""
import numpy as np
import pytest

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


def test_empty_inputs_are_noops(torch, E):
    d = 64
    P, Q = torch.ones(5, d, device='cuda'), torch.ones(7, d, device='cuda')
    z32 = torch.zeros(0, dtype=torch.int32, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_batch(P, Q, z32, z32, z32, 0.1, 0.1, 0.1, loss)
    gU, gV = torch.zeros_like(P), torch.zeros_like(Q)
    E.bpr_grad_scatter(P, Q, z32, z32, z32, 1e-7, 0.1, gU, gV, loss)
    rp0 = torch.zeros(1, dtype=torch.int64, device='cuda')
    assert E.sample_neg_philox(z32, rp0, z32, 7, 1, 1).numel() == 0
    E.gather_rows(P, z32, torch.empty(0, d, device='cuda'))
    E.scatter_add_rows(gU, z32, torch.empty(0, d, device='cuda'))
    E.sgemm(torch.empty(0, 8, device='cuda'), torch.empty(8, 4, device='cuda'), torch.empty(0, 4, device='cuda'))
    E.tc_gemm(torch.empty(0, 8, device='cuda'), torch.empty(8, 4, device='cuda'), torch.empty(0, 4, device='cuda'))
    E.adam_dense_tf1(P[:0], P[:0], P[:0], P[:0], 0.1, 1)
    E.axpby(P[:0], P[:0], P[:0], 1.0, 1.0)
    E.sumsq(P[:0], loss)
    m = __import__('qrec_b200.parallel', fromlist=['x']).ShardedItemTableBPR(P, Q, 7, 0, 1, 0.1, 0.1, 0.1)
    m.step(z32, z32, z32)
    torch.cuda.synchronize()
    assert loss.item() == 0.0 and bool((P == 1).all()) and bool((Q == 1).all()) and bool((gU == 0).all())


def test_bad_arguments_are_reported(torch, E):
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    i1 = torch.zeros(1, dtype=torch.int32, device='cuda')
    good = torch.zeros(4, 64, device='cuda')
    cases = [
        lambda: E.bpr_sgd_batch(torch.zeros(4, 260, device='cuda'), torch.zeros(4, 260, device='cuda'), i1, i1, i1, 0.1, 0, 0, loss),
        lambda: E.bpr_sgd_batch(good, good, i1.long(), i1, i1, 0.1, 0, 0, loss),               # wrong index dtype
        lambda: E.bpr_sgd_batch(good.double(), good, i1, i1, i1, 0.1, 0, 0, loss),            # wrong table dtype
        lambda: E.bpr_sgd_batch(torch.zeros(64, 8, device='cuda').t(), torch.zeros(4, 64, device='cuda'), i1, i1, i1, 0.1, 0, 0, loss),  # non-contiguous
        lambda: E.spmm_csr(torch.zeros(5, dtype=torch.int64, device='cuda'), i1, torch.zeros(1, device='cuda'), good, good),  # X aliases Y
        lambda: E.adam_dense_tf1(good, good, good, good, 0.1, 0),                              # t must be >= 1
        lambda: E.tc_gemm(torch.zeros(8, 6, device='cuda'), torch.zeros(6, 4, device='cuda'), torch.zeros(8, 4, device='cuda')),  # K % 4
        lambda: E.infonce_rows(torch.zeros(3, 3, device='cuda'), 0.0, loss),                   # tau must be > 0
        lambda: E.bpr_sgd_usermajor(good, good, torch.zeros(5, dtype=torch.int64), i1, i1, 0.1, 0, 0, loss),  # host rowptr
    ]
    for fn in cases:
        with pytest.raises(E.QRecError):
            fn()
    # the error channel carries a message
    from qrec_b200._lib import lib
    assert len(lib.qrec_last_error()) > 0


def test_widest_supported_rows(torch, E):
    """d = 256 (batch / K3 / SpMM) and d = 128 (user-major): the largest widths the kernels take."""
    from oracle import c_oracle
    rng = np.random.default_rng(0)
    for d, fn in ((256, 'batch'), (128, 'usermajor')):
        nu, ni, n = 64, 200, 64
        u = np.arange(n, dtype=np.int32)
        items = rng.permutation(ni)[:2 * n].astype(np.int32)
        i, j = items[:n].copy(), items[n:].copy()
        P0 = (rng.random((nu, d)) / 3).astype(np.float32); Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
        P, Q = torch.from_numpy(P0).cuda(), torch.from_numpy(Q0).cuda()
        loss = torch.zeros(1, dtype=torch.float64, device='cuda')
        if fn == 'batch':
            E.bpr_sgd_batch(P, Q, torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda(), torch.from_numpy(j).cuda(), 0.05, 0.01, 0.01, loss)
        else:
            rp = torch.arange(nu + 1, dtype=torch.int64, device='cuda')
            E.bpr_sgd_usermajor(P, Q, rp, torch.from_numpy(i).cuda(), torch.from_numpy(j).cuda(), 0.05, 0.01, 0.01, loss)
        Pc, Qc = P0.copy(), Q0.copy()
        c_oracle.bpr_sgd_sequential(Pc, Qc, u, i, j, 0.05, 0.01, 0.01)
        np.testing.assert_allclose(P.cpu().numpy(), Pc, rtol=2e-5, atol=1e-6)
        np.testing.assert_allclose(Q.cpu().numpy(), Qc, rtol=2e-5, atol=1e-6)
