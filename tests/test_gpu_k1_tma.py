"""qrec_bpr_epoch_usermajor_tma_f32: the fused user-major epoch with the item rows staged through shared memory by
cp.async.bulk + mbarrier (the TMA fetch of the user-major kernel body in csrc/bpr_kernels.cu).  It must draw exactly
the negatives of the stand-alone Philox sampler (bit-exact index parity) and apply the same updates as
qrec_bpr_epoch_usermajor_f32, on ragged inputs and at the benchmark learning rate."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR, REG = 0.01, 0.001          # bench.py's learning rate and regularisation


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


@pytest.mark.parametrize('nu,ni,maxdeg', [(3000, 5000, 40), (1, 300, 7), (500, 64, 20), (2000, 100000, 33)])
def test_tma_epoch_equals_ldg_epoch(torch, E, nu, ni, maxdeg):
    rng = np.random.default_rng(nu + ni)
    deg = rng.integers(0, maxdeg + 1, nu)
    if nu > 10:
        deg[3] = 0; deg[7] = 5 * maxdeg if 5 * maxdeg < ni // 2 else maxdeg           # an empty and a long user
    rowptr = np.zeros(nu + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    n = int(rowptr[-1])
    u = np.repeat(np.arange(nu), deg)
    i = np.concatenate([rng.choice(ni, k, replace=False) for k in deg] + [np.zeros(0, np.int64)]).astype(np.int32)
    csr = E.RatedCSR(nu, ni, u, i)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    P0 = (rng.random((nu, 64)) / 3).astype(np.float32); Q0 = (rng.random((ni, 64)) / 3).astype(np.float32)
    Pa, Qa, Pb, Qb = dev(P0), dev(Q0), dev(P0), dev(Q0)
    rp, ii, rrp, rc = dev(rowptr), dev(i), dev(csr.sorted_rowptr), dev(csr.sorted_cols)
    la = torch.zeros(1, dtype=torch.float64, device='cuda'); lb = torch.zeros(1, dtype=torch.float64, device='cuda')
    ja = torch.full((n,), -1, dtype=torch.int32, device='cuda'); jb = torch.full((n,), -2, dtype=torch.int32, device='cuda')
    lr, reg = 1e-4, 0.001
    E.bpr_epoch_usermajor(Pa, Qa, rp, ii, rrp, rc, ni, 0xabcdef, 3, lr, reg, reg, la, j_out=ja)
    E.bpr_epoch_usermajor_tma(Pb, Qb, rp, ii, rrp, rc, ni, 0xabcdef, 3, lr, reg, reg, lb, j_out=jb)
    torch.cuda.synchronize()
    assert torch.equal(ja, jb)
    jref = E.sample_neg_philox(dev(u.astype(np.int32)), rrp, rc, ni, 0xabcdef, 3) if n else ja
    assert torch.equal(jb, jref)
    if n == 0:
        return
    P0t, Q0t = dev(P0), dev(Q0)
    dPa, dPb, dQa, dQb = Pa - P0t, Pb - P0t, Qa - Q0t, Qb - Q0t
    assert float((dPa - dPb).abs().max()) <= 0.02 * float(dPa.abs().max())
    assert float((dQa - dQb).abs().max()) <= 0.02 * float(dQa.abs().max())
    assert abs(la.item() - lb.item()) <= 1e-4 * abs(la.item())


def test_tma_epoch_equals_ldg_epoch_at_benchmark_rate(torch, E):
    """On the schedule of test_usermajor_epoch_is_the_same_every_run (tests/test_gpu_bpr.py) the staged epoch reads
    the same wave snapshots as the LDG epoch, so the two agree up to the summation order of the scatter-adds.  A
    staged kernel that read the live item table while other lane groups added into it would miss by far more."""
    from qrec_b200 import synthetic
    dev = torch.device('cuda', 0)
    users, items, deg, d = 200_000, 20_000, 20, 64
    data = synthetic.make_interactions(users, items, deg, device=dev, seed=5)
    runs = []
    for epoch in (E.bpr_epoch_usermajor, E.bpr_epoch_usermajor_tma):
        P, Q = synthetic.init_tables(users, items, d, seed=6, device=dev)
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        epoch(P, Q, data['sorted_rowptr'], data['i'], data['sorted_rowptr'], data['sorted_cols'], items, 77, 0, LR, REG, REG,
              loss)
        torch.cuda.synchronize()
        runs.append((P.cpu(), Q.cpu(), loss.item()))
    P0, Q0 = synthetic.init_tables(users, items, d, seed=6, device=dev)
    for k, X0 in ((0, P0.cpu()), (1, Q0.cpu())):
        update = float((runs[0][k] - X0).abs().max())
        assert update > 0
        assert float((runs[0][k] - runs[1][k]).abs().max()) <= 1e-4 * update
    assert abs(runs[0][2] - runs[1][2]) <= 1e-9 * abs(runs[0][2])


def test_tma_epoch_rejects_other_widths(torch, E):
    P = torch.ones(4, 32, device='cuda'); Q = torch.ones(5, 32, device='cuda')
    rp = torch.tensor([0, 1, 2, 3, 4], dtype=torch.int64, device='cuda')
    i = torch.zeros(4, dtype=torch.int32, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    with pytest.raises(E.QRecError):
        E.bpr_epoch_usermajor_tma(P, Q, rp, i, rp, i, 5, 1, 0, 0.1, 0.1, 0.1, loss)
