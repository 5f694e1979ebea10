"""Parity tests proper for K0(fast)/K1: the CUDA path (through the C ABI) against the oracle and
the golden vectors recorded from the reference.  Needs a GPU."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR, REG = 0.01, 0.001


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _init_tables(nu, ni, d=64):
    np.random.seed(0)
    P = np.random.rand(nu, d) / 3
    Q = np.random.rand(ni, d) / 3
    return P, Q


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run_ordered(torch, E, P, Q, t, nu, ni, lr=LR, reg=REG):
    wu, wi, wj = E.bpr_order_prepare(t[:, 0], t[:, 1], t[:, 2], nu, ni)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_ordered(P, Q, _dev(torch, t[:, 0]), _dev(torch, t[:, 1]), _dev(torch, t[:, 2]),
                      _dev(torch, wu), _dev(torch, wi), _dev(torch, wj), lr, reg, reg, loss)
    torch.cuda.synchronize()
    return float(loss.item())


def test_ordered_f64_matches_reference_three_epochs(torch, E, golden_bpr, bpr_ids):
    """float64 parity mode == the reference's numpy path (model/ranking/BPR.py:19-53), incl. the
    epoch loss (BPR.py:40) and the adaptive learning rate (iterativeRecommender.py:56-63)."""
    from oracle import bpr_oracle as O
    _, _, nu, ni = bpr_ids
    P0, Q0 = _init_tables(nu, ni)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    lr, last = LR, 0.0
    for ep in range(3):
        t = golden_bpr['triples_epoch'][ep]
        loss = _run_ordered(torch, E, P, Q, t, nu, ni, lr=lr)
        reg = torch.zeros(2, dtype=torch.float64, device='cuda')
        E.sumsq(P, reg[0:1]); E.sumsq(Q, reg[1:2])
        loss += REG * float(reg[0].item()) + REG * float(reg[1].item())
        assert abs(loss - golden_bpr['loss'][ep]) <= 1e-9 * golden_bpr['loss'][ep]
        if ep == 0:
            np.testing.assert_allclose(P.cpu().numpy(), golden_bpr['P_epoch1'], rtol=1e-10, atol=1e-13)
            np.testing.assert_allclose(Q.cpu().numpy(), golden_bpr['Q_epoch1'], rtol=1e-10, atol=1e-13)
        lr = O.update_learning_rate(lr, 1.0, ep + 1, last, loss)
        assert lr == golden_bpr['lrate'][ep][1]
        last = loss
    np.testing.assert_allclose(P.cpu().numpy(), golden_bpr['P_epoch3'], rtol=2e-7, atol=1e-8)
    np.testing.assert_allclose(Q.cpu().numpy(), golden_bpr['Q_epoch3'], rtol=2e-7, atol=1e-8)


def test_ordered_f32_within_1e5_relative_after_one_epoch(torch, E, golden_bpr, bpr_ids):
    """north_star tolerance: fp32 embeddings within 1e-5 relative after one epoch (max-norm
    relative, i.e. |got-ref|_inf <= 1e-5*|ref|_inf) against the float64 reference."""
    from oracle import c_oracle
    _, _, nu, ni = bpr_ids
    P0, Q0 = _init_tables(nu, ni)
    P, Q = _dev(torch, P0.astype(np.float32)), _dev(torch, Q0.astype(np.float32))
    t = golden_bpr['triples_epoch'][0]
    loss = _run_ordered(torch, E, P, Q, t, nu, ni)
    for got, ref in ((P.cpu().numpy(), golden_bpr['P_epoch1']), (Q.cpu().numpy(), golden_bpr['Q_epoch1'])):
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()
        np.testing.assert_allclose(got, ref, rtol=1e-5, atol=2e-6)
    # and against the fp32 sequential oracle it is tighter still (same arithmetic, only the dot
    # product summation order differs)
    Pc, Qc = P0.astype(np.float32), Q0.astype(np.float32)
    closs = c_oracle.bpr_sgd_sequential(Pc, Qc, t[:, 0], t[:, 1], t[:, 2], LR, REG, REG)
    np.testing.assert_allclose(P.cpu().numpy(), Pc, rtol=2e-5, atol=2e-6)
    assert abs(loss - closs) <= 1e-5 * closs


@pytest.mark.parametrize('d', [1, 7, 50, 64, 100, 200])
def test_ordered_generic_d_heavy_conflicts(torch, E, d):
    """Few rows, many triples: almost every triple depends on its predecessor."""
    from oracle import c_oracle
    rng = np.random.default_rng(d)
    nu, ni, n = 5, 9, 3000
    u = rng.integers(0, nu, n).astype(np.int32)
    i = rng.integers(0, ni, n).astype(np.int32)
    j = ((i + 1 + rng.integers(0, ni - 1, n)) % ni).astype(np.int32)
    P0 = rng.random((nu, d)) / 3
    Q0 = rng.random((ni, d)) / 3
    t = np.stack([u, i, j], 1)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    loss = _run_ordered(torch, E, P, Q, t, nu, ni, lr=0.05, reg=0.01)
    Pc, Qc = P0.copy(), Q0.copy()
    closs = c_oracle.bpr_sgd_sequential(Pc, Qc, u, i, j, 0.05, 0.01, 0.01)
    np.testing.assert_allclose(P.cpu().numpy(), Pc, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(Q.cpu().numpy(), Qc, rtol=1e-9, atol=1e-12)
    assert abs(loss - closs) <= 1e-9 * abs(closs)


def test_ordered_empty_input(torch, E):
    P = torch.ones(3, 8, device='cuda', dtype=torch.float64)
    Q = torch.ones(4, 8, device='cuda', dtype=torch.float64)
    z = torch.zeros(0, dtype=torch.int32, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_ordered(P, Q, z, z, z, z, z, z, 0.1, 0.1, 0.1, loss)
    torch.cuda.synchronize()
    assert float(loss.item()) == 0.0 and bool((P == 1).all())


def _conflict_free_triples(rng, nu, ni, n):
    assert n <= nu and 2 * n <= ni
    u = rng.permutation(nu)[:n].astype(np.int32)
    items = rng.permutation(ni)[:2 * n].astype(np.int32)
    return u, items[:n].copy(), items[n:].copy()


@pytest.mark.parametrize('d,n', [(64, 1), (64, 31), (64, 1000), (64, 4097), (64, 70001), (16, 333), (32, 500),
                                 (48, 257), (128, 700), (256, 300), (200, 123), (8, 64)])
def test_batch_conflict_free_equals_reference_step(torch, E, d, n):
    """Triples that share no row: the fused kernel must give exactly BPR.optimization per triple
    (up to one fp32 rounding of `row + delta`)."""
    from oracle import c_oracle
    rng = np.random.default_rng(1000 * d + n)
    nu, ni = max(n, 8), max(2 * n, 16)
    u, i, j = _conflict_free_triples(rng, nu, ni, n)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32)
    Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_batch(P, Q, _dev(torch, u), _dev(torch, i), _dev(torch, j), 0.05, 0.01, 0.02, loss)
    torch.cuda.synchronize()
    Pc, Qc = P0.copy(), Q0.copy()
    closs = c_oracle.bpr_sgd_sequential(Pc, Qc, u, i, j, 0.05, 0.01, 0.02)
    np.testing.assert_allclose(P.cpu().numpy(), Pc, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(Q.cpu().numpy(), Qc, rtol=1e-6, atol=1e-7)
    assert abs(float(loss.item()) - closs) <= 1e-5 * abs(closs) + 1e-6


def test_batch_with_shared_rows_sums_deltas(torch, E):
    """Rows shared inside a launch get the SUM of per-triple deltas (scatter-add).  Reads may see
    a neighbour's delta already applied (the kernel is fused, not two-phase), which perturbs each
    delta by O(lr * |delta|); the tolerance below is that second-order term."""
    from oracle import bpr_oracle as O
    rng = np.random.default_rng(5)
    nu, ni, n, d = 50, 40, 4000, 64
    u = rng.integers(0, nu, n).astype(np.int32)
    i = rng.integers(0, ni, n).astype(np.int32)
    j = ((i + 1 + rng.integers(0, ni - 1, n)) % ni).astype(np.int32)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32)
    Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    lr = 1e-4
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_batch(P, Q, _dev(torch, u), _dev(torch, i), _dev(torch, j), lr, REG, REG, loss)
    torch.cuda.synchronize()
    dP, dQ, jl = O.bpr_sgd_jacobi(P0, Q0, np.stack([u, i, j], 1), lr, REG, REG)
    gotP = P.cpu().numpy().astype(np.float64) - P0
    gotQ = Q.cpu().numpy().astype(np.float64) - Q0
    assert np.abs(gotP - dP).max() <= 0.03 * np.abs(dP).max()
    assert np.abs(gotQ - dQ).max() <= 0.03 * np.abs(dQ).max()
    assert abs(float(loss.item()) - jl) <= 1e-3 * jl


def test_batch_bad_arguments(torch, E):
    P = torch.zeros(4, 6, device='cuda')      # d=6 not a multiple of 4
    Q = torch.zeros(4, 6, device='cuda')
    z = torch.zeros(1, dtype=torch.int32, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    with pytest.raises(E.QRecError):
        E.bpr_sgd_batch(P, Q, z, z, z, 0.1, 0, 0, loss)
    with pytest.raises(E.QRecError):          # CPU tensors are rejected: there is no CPU path
        E.bpr_sgd_batch(P.cpu(), Q, z, z, z, 0.1, 0, 0, loss)


def test_batch_training_tracks_sequential_loss_curve(torch, E, golden_bpr, bpr_ids):
    """Throughput mode on the reference's own FilmTrust triples, launched in minibatches of 1024
    (on a table this small a single launch would hold the whole epoch in flight at once, i.e. be
    a Jacobi step over the epoch): the epoch losses follow the reference's Gauss-Seidel curve."""
    _, _, nu, ni = bpr_ids
    P0, Q0 = _init_tables(nu, ni)
    P, Q = _dev(torch, P0.astype(np.float32)), _dev(torch, Q0.astype(np.float32))
    rng = np.random.default_rng(0)
    for ep in range(3):
        t = golden_bpr['triples_epoch'][ep][rng.permutation(golden_bpr['triples_epoch'].shape[1])]
        tu, ti, tj = (_dev(torch, t[:, c]) for c in range(3))
        lr = float(golden_bpr['lrate'][ep][0])
        loss = torch.zeros(3, dtype=torch.float64, device='cuda')
        for b in range(0, len(t), 1024):
            E.bpr_sgd_batch(P, Q, tu[b:b + 1024], ti[b:b + 1024], tj[b:b + 1024], lr, REG, REG, loss[0:1])
        E.sumsq(P, loss[1:2]); E.sumsq(Q, loss[2:3])
        l = loss.cpu().numpy()
        total = l[0] + REG * l[1] + REG * l[2]
        assert abs(total - golden_bpr['loss'][ep]) <= 0.05 * golden_bpr['loss'][ep]


def test_host_pipeline_equals_device_call(torch, E):
    rng = np.random.default_rng(11)
    nu, ni, n, d = 5000, 9000, 3000, 64
    u, i, j = _conflict_free_triples(rng, nu, ni, n)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32)
    Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    Pa, Qa, Pb, Qb = _dev(torch, P0), _dev(torch, Q0), _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_batch(Pa, Qa, _dev(torch, u), _dev(torch, i), _dev(torch, j), 0.05, 0.01, 0.01, loss)
    pipe = E.HostPipeline(0, chunk_triples=700)       # 5 chunks, last one short
    hu, hi, hj = (torch.from_numpy(x).pin_memory() for x in (u, i, j))
    hl = pipe.bpr_epoch(Pb, Qb, hu, hi, hj, 0.05, 0.01, 0.01)
    torch.cuda.synchronize()
    assert torch.equal(Pa, Pb) and torch.equal(Qa, Qb)
    assert abs(hl - float(loss.item())) <= 1e-6 * abs(hl)      # fp32 partial sums regroup per chunk
    # pageable numpy input and an empty epoch
    assert pipe.bpr_epoch(Pb, Qb, u[:0].copy(), i[:0].copy(), j[:0].copy(), 0.05, 0.01, 0.01) == 0.0
    pipe.close()


def test_philox_sampler_bit_exact_and_valid(torch, E, bpr_ids):
    from oracle import bpr_oracle as O
    from conftest import rows_and_sets
    u, i, nu, ni = bpr_ids
    csr = E.RatedCSR(nu, ni, u, i)
    _, sets = rows_and_sets(u, i, nu)
    rp, cols = _dev(torch, csr.sorted_rowptr), _dev(torch, csr.sorted_cols)
    for seed, epoch in ((0, 0), (0x1234567890abcdef, 3)):
        j = E.sample_neg_philox(_dev(torch, u), rp, cols, ni, seed, epoch).cpu().numpy()
        ref = O.sample_neg_philox(u.tolist(), sets, ni, seed, epoch)
        assert np.array_equal(j, ref)
        assert all(jj not in sets[uu] for uu, jj in zip(u.tolist(), j.tolist()))
        assert j.min() >= 0 and j.max() < ni
    # dense user: 1890 of 1891 items rated -> many rejections, still terminates and is exact
    dense_items = np.arange(ni - 1)
    csr2 = E.RatedCSR(1, ni, np.zeros(ni - 1, np.int64), dense_items)
    uu = torch.zeros(257, dtype=torch.int32, device='cuda')
    j2 = E.sample_neg_philox(uu, _dev(torch, csr2.sorted_rowptr), _dev(torch, csr2.sorted_cols), ni, 9, 1)
    assert bool((j2 == ni - 1).all())
    # a user that rated EVERY item has no negative: the kernel returns the first draw instead of hanging
    csr3 = E.RatedCSR(1, 37, np.zeros(37, np.int64), np.arange(37))
    j3 = E.sample_neg_philox(torch.zeros(100, dtype=torch.int32, device='cuda'), _dev(torch, csr3.sorted_rowptr),
                             _dev(torch, csr3.sorted_cols), 37, 3, 0)
    torch.cuda.synchronize()
    assert int(j3.min()) >= 0 and int(j3.max()) < 37


def test_sumsq(torch, E):
    rng = np.random.default_rng(2)
    for n in (1, 3, 4, 1027, 1 << 20):
        x = rng.standard_normal(n)
        for dt in (np.float32, np.float64):
            xs = x.astype(dt)
            out = torch.zeros(1, dtype=torch.float64, device='cuda')
            E.sumsq(_dev(torch, xs), out)
            ref = float((xs.astype(np.float64) ** 2).sum())
            assert abs(float(out.item()) - ref) <= 1e-12 * ref + 1e-300


def test_full_size_properties_synthetic(torch, E):
    """BASELINE-size tables (1M x 100K, d=64), 4M shuffled triples: size-independent properties.
    (1) lr=0 with reg=0 is the identity; (2) rows not named by any triple are untouched;
    (3) the loss equals sum softplus(-x) computed by an independent torch expression."""
    g = torch.Generator(device='cuda'); g.manual_seed(1)
    nu, ni, d, n = 1_000_000, 100_000, 64, 1 << 22
    P = torch.rand(nu, d, device='cuda', generator=g) / 3
    Q = torch.rand(ni, d, device='cuda', generator=g) / 3
    u = torch.randint(0, nu // 2, (n,), device='cuda', generator=g, dtype=torch.int32)   # upper half never touched
    i = torch.randint(0, ni // 2, (n,), device='cuda', generator=g, dtype=torch.int32)
    j = torch.randint(ni // 2, ni - 1000, (n,), device='cuda', generator=g, dtype=torch.int32)
    P0, Q0 = P.clone(), Q.clone()
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_batch(P, Q, u, i, j, 0.0, 0.0, 0.0, loss)
    assert torch.equal(P, P0) and torch.equal(Q, Q0)
    ul, il, jl = u.long(), i.long(), j.long()
    x = (P0[ul] * (Q0[il] - Q0[jl])).sum(1).double()
    ref = torch.nn.functional.softplus(-x).sum().item()
    assert abs(loss.item() - ref) <= 1e-5 * ref
    E.bpr_sgd_batch(P, Q, u, i, j, 0.01, 0.001, 0.001, loss)
    torch.cuda.synchronize()
    assert torch.equal(P[nu // 2:], P0[nu // 2:]) and torch.equal(Q[ni - 1000:], Q0[ni - 1000:])
    assert not torch.equal(P[:nu // 2], P0[:nu // 2])
    assert bool(torch.isfinite(P).all()) and bool(torch.isfinite(Q).all())


def test_sharded_item_table_path_single_rank_equals_batch_kernel(torch, E):
    """K7 with world=1: ids -> owner gather -> staged K1 -> delta scatter-add must reproduce the
    fused batch kernel (conflict-free batch, so both equal the reference step)."""
    from qrec_b200 import parallel
    rng = np.random.default_rng(21)
    nu, ni, n, d = 3000, 5000, 2500, 64
    u, i, j = _conflict_free_triples(rng, nu, ni, n)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32)
    Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    Pa, Qa, Pb, Qb = _dev(torch, P0), _dev(torch, Q0), _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_batch(Pa, Qa, _dev(torch, u), _dev(torch, i), _dev(torch, j), 0.05, 0.01, 0.02, loss)
    m = parallel.ShardedItemTableBPR(Pb, Qb, ni, 0, 1, 0.05, 0.01, 0.02)
    l2 = m.step(_dev(torch, u), _dev(torch, i), _dev(torch, j))
    torch.cuda.synchronize()
    torch.testing.assert_close(Pb, Pa, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(Qb, Qa, rtol=1e-6, atol=1e-7)
    assert abs(l2.item() - loss.item()) <= 1e-6 * abs(loss.item())
    # duplicates: the same item requested many times -> deltas sum at the owner
    u2 = np.arange(64, dtype=np.int32); i2 = np.full(64, 7, np.int32); j2 = np.full(64, 9, np.int32)
    Pc, Qc = _dev(torch, P0), _dev(torch, Q0)
    m2 = parallel.ShardedItemTableBPR(Pc, Qc, ni, 0, 1, 1e-3, 0.0, 0.0)
    m2.step(_dev(torch, u2), _dev(torch, i2), _dev(torch, j2))
    from oracle import bpr_oracle as O
    dP, dQ, _ = O.bpr_sgd_jacobi(P0, Q0, np.stack([u2, i2, j2], 1), 1e-3, 0.0, 0.0)
    np.testing.assert_allclose(Qc.cpu().numpy()[[7, 9]] - Q0[[7, 9]], dQ[[7, 9]], rtol=1e-3, atol=1e-7)


def _user_major_problem(rng, nu, ni, max_deg, distinct_items=True):
    if distinct_items:
        deg = np.where(rng.random(nu) < 0.1, 0, max_deg)     # chunk-aligned users, some empty
    else:
        deg = rng.integers(0, max_deg + 1, nu)
        deg[rng.integers(0, nu, 3)] = 0                   # some empty users
        deg[0] = 3 * max_deg                              # one user spanning several chunks
    rowptr = np.zeros(nu + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    n = int(rowptr[-1])
    if distinct_items:
        assert 2 * n <= ni
        items = rng.permutation(ni)[:2 * n].astype(np.int32)
        i, j = items[:n].copy(), items[n:].copy()
    else:
        i = rng.integers(0, ni, n).astype(np.int32)
        j = ((i + 1 + rng.integers(0, ni - 1, n)) % ni).astype(np.int32)
    u = np.repeat(np.arange(nu), deg).astype(np.int32)
    return rowptr, u, i, j


@pytest.mark.parametrize('d', [64, 32, 48, 128, 16])
def test_usermajor_kernel_is_sequential_in_P(torch, E, d):
    """User-major kernel: P[u] lives in registers across the triples of a user that fall into one
    32-triple chunk, so with globally distinct items and users aligned to chunks (here: every user
    has exactly 32 or 0 triples) the result must equal the SEQUENTIAL reference loop (BPR.py:31-39)."""
    from oracle import c_oracle
    rng = np.random.default_rng(d)
    nu, max_deg = 300, 32
    rowptr, u, i, j = _user_major_problem(rng, nu, 60000, max_deg)
    ni = 60000
    P0 = (rng.random((nu, d)) / 3).astype(np.float32)
    Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_usermajor(P, Q, _dev(torch, rowptr), _dev(torch, i), _dev(torch, j), 0.05, 0.01, 0.02, loss)
    torch.cuda.synchronize()
    Pc, Qc = P0.copy(), Q0.copy()
    closs = c_oracle.bpr_sgd_sequential(Pc, Qc, u, i, j, 0.05, 0.01, 0.02)
    np.testing.assert_allclose(P.cpu().numpy(), Pc, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(Q.cpu().numpy(), Qc, rtol=2e-5, atol=2e-6)
    assert abs(float(loss.item()) - closs) <= 1e-5 * abs(closs)


def test_usermajor_kernel_shared_items_and_reference_epoch(torch, E, golden_bpr, bpr_ids):
    """(a) items shared between users: Q receives the atomic sum of deltas (second-order close to the
    Jacobi restatement at small lr); (b) the reference's own first-epoch stream (user-major by
    construction) in one launch tracks the reference's epoch loss far better than a shuffled launch."""
    from oracle import bpr_oracle as O
    rng = np.random.default_rng(77)
    nu, ni, d = 200, 150, 64
    rowptr, u, i, j = _user_major_problem(rng, nu, ni, 30, distinct_items=False)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32)
    Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    P, Q = _dev(torch, P0), _dev(torch, Q0)
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_sgd_usermajor(P, Q, _dev(torch, rowptr), _dev(torch, i), _dev(torch, j), 1e-4, REG, REG, loss)
    torch.cuda.synchronize()
    dP, dQ, jl = O.bpr_sgd_jacobi(P0, Q0, np.stack([u, i, j], 1), 1e-4, REG, REG)
    assert np.abs(P.cpu().numpy().astype(np.float64) - P0 - dP).max() <= 0.03 * np.abs(dP).max()
    assert np.abs(Q.cpu().numpy().astype(np.float64) - Q0 - dQ).max() <= 0.03 * np.abs(dQ).max()
    assert abs(loss.item() - jl) <= 1e-3 * jl
    # (b)
    _, _, nu, ni = bpr_ids
    P0, Q0 = _init_tables(nu, ni)
    t = golden_bpr['triples_epoch'][0]
    assert np.all(np.diff(t[:, 0]) >= 0)                               # the reference stream is user-major
    rp = np.zeros(nu + 1, np.int64); np.add.at(rp, t[:, 0] + 1, 1); rp = np.cumsum(rp)
    P, Q = _dev(torch, P0.astype(np.float32)), _dev(torch, Q0.astype(np.float32))
    acc = torch.zeros(3, dtype=torch.float64, device='cuda')
    E.bpr_sgd_usermajor(P, Q, _dev(torch, rp), _dev(torch, t[:, 1]), _dev(torch, t[:, 2]), LR, REG, REG, acc[0:1])
    E.sumsq(P, acc[1:2]); E.sumsq(Q, acc[2:3])
    a = acc.cpu().numpy()
    total = a[0] + REG * (a[1] + a[2])
    assert abs(total - golden_bpr['loss'][0]) <= 0.06 * golden_bpr['loss'][0]


def test_usermajor_empty_and_bad_args(torch, E):
    P, Q = torch.ones(4, 64, device='cuda'), torch.ones(5, 64, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    z = torch.zeros(0, dtype=torch.int32, device='cuda')
    E.bpr_sgd_usermajor(P, Q, torch.zeros(5, dtype=torch.int64, device='cuda'), z, z, 0.1, 0.1, 0.1, loss)
    torch.cuda.synchronize()
    assert bool((P == 1).all()) and loss.item() == 0.0
    with pytest.raises(E.QRecError):
        E.bpr_sgd_usermajor(torch.ones(4, 200, device='cuda'), torch.ones(5, 200, device='cuda'),
                            torch.zeros(5, dtype=torch.int64, device='cuda'), z, z, 0.1, 0.1, 0.1, loss)


def test_usermajor_epoch_is_the_same_every_run(torch, E):
    """Two fused epochs from the same tables and stream agree up to the summation order of the scatter-adds: what a
    triple reads does not depend on timing (each user whole in one lane group; item rows read from the snapshot of
    the wave).  Reads that raced with other lane groups' scatter-adds made runs differ by a fifth of the update."""
    from qrec_b200 import synthetic
    dev = torch.device('cuda', 0)
    users, items, deg, d = 200_000, 20_000, 20, 64
    data = synthetic.make_interactions(users, items, deg, device=dev, seed=5)
    sig = E.rated_signature(data['sorted_rowptr'], data['sorted_cols'])
    runs = []
    for _ in range(2):
        P, Q = synthetic.init_tables(users, items, d, seed=6, device=dev)
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        E.bpr_epoch_usermajor_sig(P, Q, data['sorted_rowptr'], data['i'], data['sorted_rowptr'], data['sorted_cols'], sig,
                                  items, 77, 0, LR, REG, REG, loss)
        torch.cuda.synchronize()
        runs.append((P.cpu(), Q.cpu(), loss.item()))
    P0, Q0 = synthetic.init_tables(users, items, d, seed=6, device=dev)
    for k, X0 in ((0, P0.cpu()), (1, Q0.cpu())):
        update = float((runs[0][k] - X0).abs().max())
        assert update > 0
        assert float((runs[0][k] - runs[1][k]).abs().max()) <= 1e-4 * update
    assert abs(runs[0][2] - runs[1][2]) <= 1e-9 * abs(runs[0][2])


def test_fused_epoch_equals_sampler_plus_kernel(torch, E, bpr_ids):
    """qrec_bpr_epoch_usermajor_f32 (sampling fused into the user-major kernel) draws exactly the
    negatives qrec_sample_neg_philox draws (same Philox counters) and then does the same updates."""
    u, i, nu, ni = bpr_ids
    csr = E.RatedCSR(nu, ni, u, i)
    # CSR order of the positives = the reference's iteration order
    cu = np.repeat(np.arange(nu), np.diff(csr.pos_rowptr)).astype(np.int32)
    ci = csr.pos_cols
    P0, Q0 = _init_tables(nu, ni)
    Pa, Qa = _dev(torch, P0.astype(np.float32)), _dev(torch, Q0.astype(np.float32))
    Pb, Qb = Pa.clone(), Qa.clone()
    rp, rrp, rc = _dev(torch, csr.pos_rowptr), _dev(torch, csr.sorted_rowptr), _dev(torch, csr.sorted_cols)
    la = torch.zeros(1, dtype=torch.float64, device='cuda'); lb = torch.zeros(1, dtype=torch.float64, device='cuda')
    lr = 1e-4
    j_ref = E.sample_neg_philox(_dev(torch, cu), rrp, rc, ni, 0xfeedface, 5)
    E.bpr_sgd_usermajor(Pa, Qa, rp, _dev(torch, ci), j_ref, lr, REG, REG, la)
    j_out = torch.full_like(j_ref, -1)
    E.bpr_epoch_usermajor(Pb, Qb, rp, _dev(torch, ci), rrp, rc, ni, 0xfeedface, 5, lr, REG, REG, lb, j_out=j_out)
    torch.cuda.synchronize()
    assert torch.equal(j_out, j_ref)                                     # the sampled stream is bit-identical
    # the whole FilmTrust epoch is in flight at once and items are shared by hundreds of triples, so
    # the two launches interleave their item-row reads differently (second order in lr): compare
    # the applied updates, not the bits
    P0t, Q0t = _dev(torch, P0.astype(np.float32)), _dev(torch, Q0.astype(np.float32))
    dPa, dPb, dQa, dQb = Pa - P0t, Pb - P0t, Qa - Q0t, Qb - Q0t
    assert float((dPa - dPb).abs().max()) <= 0.02 * float(dPa.abs().max())
    assert float((dQa - dQb).abs().max()) <= 0.02 * float(dQa.abs().max())
    assert abs(la.item() - lb.item()) <= 1e-4 * abs(la.item())
    # without j_out, and a different epoch gives different negatives
    E.bpr_epoch_usermajor(Pb, Qb, rp, _dev(torch, ci), rrp, rc, ni, 0xfeedface, 6, lr, REG, REG, lb)
    j6 = E.sample_neg_philox(_dev(torch, cu), rrp, rc, ni, 0xfeedface, 6)
    assert not torch.equal(j6, j_ref)


def test_usermajor_host_pipeline_matches_single_launch(torch, E):
    """qrec_bpr_epoch_usermajor_host: positives in HOST memory, chunks of whole users staged while the
    fused kernel runs; Philox counters are global, so the negatives (and, up to the order in which item
    deltas land, the tables) equal the single-launch fused epoch whatever the chunking."""
    rng = np.random.default_rng(31)
    nu, ni, d = 4000, 50000, 64
    deg = rng.integers(0, 40, nu); deg[5] = 0; deg[17] = 300
    rowptr = np.zeros(nu + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    n = int(rowptr[-1])
    u = np.repeat(np.arange(nu), deg)
    i = rng.integers(0, ni, n).astype(np.int32)
    csr = E.RatedCSR(nu, ni, u, i)
    P0 = (rng.random((nu, d)) / 3).astype(np.float32); Q0 = (rng.random((ni, d)) / 3).astype(np.float32)
    Pa, Qa, Pb, Qb = _dev(torch, P0), _dev(torch, Q0), _dev(torch, P0), _dev(torch, Q0)
    rrp, rc = _dev(torch, csr.sorted_rowptr), _dev(torch, csr.sorted_cols)
    la = torch.zeros(1, dtype=torch.float64, device='cuda')
    lr = 1e-3
    E.bpr_epoch_usermajor(Pa, Qa, _dev(torch, rowptr), _dev(torch, i), rrp, rc, ni, 77, 2, lr, REG, REG, la)
    pipe = E.HostPipeline(0, chunk_triples=5000)                    # ~16 chunks, one holds the 300-triple user
    hl = pipe.bpr_epoch_usermajor(Pb, Qb, torch.from_numpy(rowptr).pin_memory(), torch.from_numpy(i).pin_memory(),
                                  rrp, rc, ni, 77, 2, lr, REG, REG)
    torch.cuda.synchronize()
    P0t, Q0t = _dev(torch, P0), _dev(torch, Q0)
    assert float(((Pa - P0t) - (Pb - P0t)).abs().max()) <= 0.02 * float((Pa - P0t).abs().max())
    assert float(((Qa - Q0t) - (Qb - Q0t)).abs().max()) <= 0.02 * float((Qa - Q0t).abs().max())
    assert abs(hl - la.item()) <= 1e-4 * abs(hl)
    # the same pipeline with the rated-set signatures attached: identical negatives, so the same loss and tables
    Pc, Qc = _dev(torch, P0), _dev(torch, Q0)
    pipe.set_rated_signature(E.rated_signature(rrp, rc))
    hl_sig = pipe.bpr_epoch_usermajor(Pc, Qc, torch.from_numpy(rowptr).pin_memory(), torch.from_numpy(i).pin_memory(),
                                      rrp, rc, ni, 77, 2, lr, REG, REG)
    pipe.set_rated_signature(None)
    torch.cuda.synchronize()
    assert abs(hl_sig - hl) <= 1e-4 * abs(hl)
    assert float(((Pc - P0t) - (Pb - P0t)).abs().max()) <= 0.02 * float((Pb - P0t).abs().max())
    # a user with more positives than the staging chunk is reported, not silently split
    small = E.HostPipeline(0, chunk_triples=100)
    with pytest.raises(E.QRecError):
        small.bpr_epoch_usermajor(Pb, Qb, rowptr, i, rrp, rc, ni, 77, 2, lr, REG, REG)
    small.close(); pipe.close()
