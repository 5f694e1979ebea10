"""Parity tests for K2 (SpMM), K3 (BPR gradient scatter), K4 (TF1 Adam) and the composed
LightGCN step, against the oracle restatements and the reference's own adjacency.  Needs a GPU."""
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


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _golden_adj(g):
    import scipy.sparse as sp
    return sp.csr_matrix((g['adj_data'], g['adj_indices'], g['adj_indptr']), shape=tuple(g['adj_shape']))


@pytest.mark.parametrize('rowsplit', [False, True])
@pytest.mark.parametrize('d', [64, 16, 32, 48, 128, 256, 8])
def test_spmm_reference_adjacency(torch, E, golden_graph, d, rowsplit):
    adj = _golden_adj(golden_graph)
    rng = np.random.default_rng(d)
    X = rng.standard_normal((adj.shape[0], d)).astype(np.float32)
    Y = torch.empty(adj.shape[0], d, device='cuda')
    acc0 = rng.standard_normal((adj.shape[0], d)).astype(np.float32)
    acc = _dev(torch, acc0)
    E.spmm_csr(_dev(torch, adj.indptr.astype(np.int64)), _dev(torch, adj.indices), _dev(torch, adj.data),
               _dev(torch, X), Y, acc=acc, acc_scale=0.25, rowsplit=rowsplit)
    ref = (adj.astype(np.float64) @ X.astype(np.float64))
    np.testing.assert_allclose(Y.cpu().numpy(), ref, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(acc.cpu().numpy(), acc0 + 0.25 * ref, rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize('rowsplit', [False, True])
def test_spmm_ragged_rows(torch, E, rowsplit):
    """Empty rows, a single huge row, rows longer than one lane-group chunk, and a row ending at every gather-batch and
    index-chunk boundary of the d = 64 row-split kernel (8 gathers per batch, 16 entries per chunk)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(3)
    n, m, d = 300, 600, 64
    rows, cols = [], []
    for r in range(n):
        deg = 0 if r % 7 == 0 else (n if r == 5 else int(rng.integers(1, 40)))
        c = rng.choice(n, size=deg, replace=False)
        rows += [r] * deg; cols += c.tolist()
    boundary = (1, 3, 4, 5, 8, 9, 15, 16, 17, 31, 32, 33, 0, 600)
    for k, deg in enumerate(boundary):
        rows += [n + k] * deg; cols += rng.choice(m, size=deg, replace=False).tolist()
    nr = n + len(boundary)
    A = sp.csr_matrix((rng.standard_normal(len(rows)).astype(np.float32), (rows, cols)), shape=(nr, m))
    A.sort_indices()
    X = rng.standard_normal((m, d)).astype(np.float32)
    Y = torch.full((nr, d), 7.0, device='cuda')
    E.spmm_csr(_dev(torch, A.indptr.astype(np.int64)), _dev(torch, A.indices), _dev(torch, A.data), _dev(torch, X), Y,
               rowsplit=rowsplit)
    np.testing.assert_allclose(Y.cpu().numpy(), A.astype(np.float64) @ X, rtol=1e-4, atol=1e-5)
    assert bool((Y[0] == 0).all()) and bool((Y[n + 12] == 0).all())    # empty rows are written as zeros, not left stale


def test_spmm_power_law_rows_split_across_chunks(torch, E):
    """A few rows far longer than the 1024-nnz chunk (hot items), many empty rows at both ends, and
    the fused accumulate on rows that straddle chunk boundaries."""
    import scipy.sparse as sp
    rng = np.random.default_rng(9)
    n, d = 4000, 64
    deg = np.minimum((n * rng.random(n) ** 6).astype(int), n)
    deg[:5] = 0; deg[-7:] = 0; deg[10] = 3000; deg[11] = 1; deg[12] = 2500
    rows = np.repeat(np.arange(n), deg)
    cols = np.concatenate([rng.choice(n, k, replace=False) for k in deg if k > 0])
    A = sp.csr_matrix((rng.standard_normal(len(rows)).astype(np.float32), (rows, cols)), shape=(n, n))
    A.sort_indices()
    X = rng.standard_normal((n, d)).astype(np.float32)
    acc0 = rng.standard_normal((n, d)).astype(np.float32)
    ref = A.astype(np.float64) @ X.astype(np.float64)
    for rowsplit in (False, True):
        Y = torch.full((n, d), 3.0, device='cuda')
        acc = _dev(torch, acc0)
        E.spmm_csr(_dev(torch, A.indptr.astype(np.int64)), _dev(torch, A.indices), _dev(torch, A.data),
                   _dev(torch, X), Y, acc=acc, acc_scale=-0.5, rowsplit=rowsplit)
        # rows of up to 3000 unit-variance terms: fp32 accumulation error ~ 1e-4 absolute
        np.testing.assert_allclose(Y.cpu().numpy(), ref, rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(acc.cpu().numpy(), acc0 - 0.5 * ref, rtol=1e-3, atol=1e-3)
    # all-empty matrix
    Z = sp.csr_matrix((n, n), dtype=np.float32)
    Y = torch.full((n, d), 3.0, device='cuda')
    E.spmm_csr(_dev(torch, Z.indptr.astype(np.int64)), _dev(torch, Z.indices.astype(np.int32)),
               _dev(torch, Z.data), _dev(torch, X), Y)
    assert bool((Y == 0).all())


def test_spmm_symmetric_linear(torch, E, golden_graph):
    """Properties the backward pass relies on: A is symmetric, so <A x, y> = <x, A y>; linearity."""
    adj = _golden_adj(golden_graph)
    rp, ci, va = _dev(torch, adj.indptr.astype(np.int64)), _dev(torch, adj.indices), _dev(torch, adj.data)
    g = torch.Generator(device='cuda'); g.manual_seed(0)
    x = torch.randn(adj.shape[0], 64, device='cuda', generator=g)
    y = torch.randn(adj.shape[0], 64, device='cuda', generator=g)
    Ax, Ay, Axy = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    E.spmm_csr(rp, ci, va, x, Ax); E.spmm_csr(rp, ci, va, y, Ay); E.spmm_csr(rp, ci, va, 2 * x - 3 * y, Axy)
    a, b = (Ax.double() * y.double()).sum().item(), (x.double() * Ay.double()).sum().item()
    assert abs(a - b) <= 1e-5 * max(abs(a), 1.0)
    torch.testing.assert_close(Axy, 2 * Ax - 3 * Ay, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize('d,n', [(64, 2048), (64, 1), (64, 1669), (32, 300), (128, 500), (256, 100)])
def test_bpr_grad_scatter(torch, E, d, n):
    from oracle import bpr_oracle as O
    rng = np.random.default_rng(d + n)
    nu, ni = 200, 150                     # small tables -> many duplicate indices inside the batch
    U = (rng.standard_normal((nu, d)) * 0.1).astype(np.float32)
    V = (rng.standard_normal((ni, d)) * 0.1).astype(np.float32)
    u = rng.integers(0, nu, n).astype(np.int32)
    i = rng.integers(0, ni, n).astype(np.int32)
    j = rng.integers(0, ni, n).astype(np.int32)
    gU, gV = torch.zeros(nu, d, device='cuda'), torch.zeros(ni, d, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_grad_scatter(_dev(torch, U), _dev(torch, V), _dev(torch, u), _dev(torch, i), _dev(torch, j),
                       1e-7, 0.001, gU, gV, loss)
    rl, rU, rV = O.bpr_loss_grad(U, V, u, i, j, 1e-7, 0.001)
    np.testing.assert_allclose(gU.cpu().numpy(), rU, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(gV.cpu().numpy(), rV, rtol=1e-4, atol=1e-6)
    assert abs(loss.item() - rl) <= 1e-5 * abs(rl)


def test_bpr_grad_matches_torch_autograd(torch, E):
    """Independent check of the hand-derived gradient (util/loss.py:3-6 + batch L2)."""
    g = torch.Generator(device='cuda'); g.manual_seed(4)
    nu, ni, d, n = 64, 80, 64, 512
    U = (torch.randn(nu, d, device='cuda', generator=g) * 0.2).requires_grad_()
    V = (torch.randn(ni, d, device='cuda', generator=g) * 0.2).requires_grad_()
    u = torch.randint(0, nu, (n,), device='cuda', generator=g)
    i = torch.randint(0, ni, (n,), device='cuda', generator=g)
    j = torch.randint(0, ni, (n,), device='cuda', generator=g)
    ue, pe, ne = U[u], V[i], V[j]
    score = (ue * pe).sum(1) - (ue * ne).sum(1)
    l = -torch.log(torch.sigmoid(score) + 10e-8).sum() + 0.001 * 0.5 * ((ue ** 2).sum() + (pe ** 2).sum() + (ne ** 2).sum())
    l.backward()
    gU, gV = torch.zeros(nu, d, device='cuda'), torch.zeros(ni, d, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_grad_scatter(U.detach(), V.detach(), u.int(), i.int(), j.int(), 10e-8, 0.001, gU, gV, loss)
    torch.testing.assert_close(gU, U.grad, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(gV, V.grad, rtol=1e-4, atol=1e-6)
    assert abs(loss.item() - l.item()) <= 1e-5 * abs(l.item())


def test_adam_tf1(torch, E):
    from oracle import bpr_oracle as O
    rng = np.random.default_rng(8)
    for n in (5, 4096, 64 * 1001 + 3):
        var = rng.standard_normal(n).astype(np.float32)
        m = np.zeros(n, np.float32); v = np.zeros(n, np.float32)
        dv, dm, dvv = _dev(torch, var), _dev(torch, m), _dev(torch, v)
        for t in range(1, 6):
            g = (rng.standard_normal(n) * (t % 2)).astype(np.float32)   # zero grads still move var (dense Adam)
            O.adam_tf1(var, m, v, g, 0.001, t)
            E.adam_dense_tf1(dv, dm, dvv, _dev(torch, g), 0.001, t)
        np.testing.assert_allclose(dv.cpu().numpy(), var, rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(dm.cpu().numpy(), m, rtol=1e-5, atol=1e-7)   # fma vs mul+add near 0
        np.testing.assert_allclose(dvv.cpu().numpy(), v, rtol=1e-5, atol=1e-9)
        # the variant that reads the step factor from device memory (for CUDA-graph replays) returns the same bits
        a = [t_.clone() for t_ in (dv, dm, dvv)]
        b = [t_.clone() for t_ in (dv, dm, dvv)]
        gg = _dev(torch, rng.standard_normal(n).astype(np.float32))
        E.adam_dense_tf1(a[0], a[1], a[2], gg, 0.001, 7)
        E.adam_dense_tf1_devstep(b[0], b[1], b[2], gg, torch.tensor([E.adam_lr_t(0.001, 7)], dtype=torch.float32, device='cuda'))
        assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_spmm_scatter_rows_equals_dense_product(torch, E, golden_graph):
    """First-backward shortcut: X non-zero only in a few rows -> scatter along those rows' edges."""
    adj = _golden_adj(golden_graph)
    n, d = adj.shape[0], 64
    rng = np.random.default_rng(4)
    nz = np.unique(rng.integers(0, n, 700)).astype(np.int32)
    nz = np.concatenate([nz, np.array([int(np.argmax(np.diff(adj.indptr)))], np.int32)])     # + the longest row
    nz = np.unique(nz)
    X = np.zeros((n, d), np.float32)
    X[nz] = rng.standard_normal((len(nz), d)).astype(np.float32)
    acc0 = rng.standard_normal((n, d)).astype(np.float32)
    acc = _dev(torch, acc0)
    Y = torch.full((n, d), 5.0, device='cuda')
    E.spmm_csr_scatter_rows(_dev(torch, adj.indptr.astype(np.int64)), _dev(torch, adj.indices), _dev(torch, adj.data),
                            _dev(torch, nz), _dev(torch, X), Y, acc=acc, acc_scale=0.25)
    ref = adj.astype(np.float64) @ X.astype(np.float64)
    np.testing.assert_allclose(Y.cpu().numpy(), ref, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(acc.cpu().numpy(), acc0 + 0.25 * ref, rtol=1e-4, atol=1e-6)
    # no source rows: Y is just zero-filled
    E.spmm_csr_scatter_rows(_dev(torch, adj.indptr.astype(np.int64)), _dev(torch, adj.indices), _dev(torch, adj.data),
                            torch.zeros(0, dtype=torch.int32, device='cuda'), _dev(torch, X), Y)
    assert bool((Y == 0).all())


@pytest.mark.parametrize('d', [8, 32, 52, 64, 128])
def test_spmm_listed_rows_equals_dense_product(torch, E, golden_graph, d):
    """Last-forward shortcut: only a list of output rows of A @ X (one warp per row, lane groups splitting the
    row's entries).  Direct, compact and accumulate-only outputs; -1 entries are padding; unlisted rows untouched."""
    adj = _golden_adj(golden_graph)
    n = adj.shape[0]
    rng = np.random.default_rng(14)
    rows = np.unique(rng.integers(0, n, 600)).astype(np.int32)
    rows = np.unique(np.concatenate([rows, [int(np.argmax(np.diff(adj.indptr)))],       # the longest row
                                     [int(np.argmin(np.diff(adj.indptr)))]])).astype(np.int32)   # and a shortest one
    padded = np.full(len(rows) + 37, -1, np.int32)
    slots = np.sort(rng.choice(len(padded), len(rows), replace=False))
    padded[slots] = rows
    X = rng.standard_normal((n, d)).astype(np.float32)
    ref = (adj.astype(np.float64) @ X.astype(np.float64))
    csr = (_dev(torch, adj.indptr.astype(np.int64)), _dev(torch, adj.indices), _dev(torch, adj.data))
    dX, dr = _dev(torch, X), _dev(torch, padded)
    # rows of a full-height output + accumulation
    acc0 = rng.standard_normal((n, d)).astype(np.float32)
    acc, Y = _dev(torch, acc0), torch.full((n, d), 7.0, device='cuda')
    E.spmm_csr_rows(*csr, dr, dX, Y, acc=acc, acc_scale=0.25)
    got, gacc = Y.cpu().numpy(), acc.cpu().numpy()
    np.testing.assert_allclose(got[rows], ref[rows], rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(gacc[rows], acc0[rows] + 0.25 * ref[rows], rtol=1e-4, atol=2e-6)
    other = np.setdiff1d(np.arange(n), rows)
    assert np.all(got[other] == 7.0) and np.array_equal(gacc[other], acc0[other])
    # compact output: row k of Y belongs to list entry k, padding entries give zero rows
    Yc = torch.full((len(padded), d), 7.0, device='cuda')
    E.spmm_csr_rows(*csr, dr, dX, Yc, compact=True)
    gc = Yc.cpu().numpy()
    np.testing.assert_allclose(gc[slots], ref[rows], rtol=1e-4, atol=2e-6)
    assert np.all(gc[padded < 0] == 0.0)
    # accumulate only; twice the same call is deterministic
    a1, a2 = _dev(torch, acc0), _dev(torch, acc0)
    E.spmm_csr_rows(*csr, dr, dX, None, acc=a1, acc_scale=-1.5)
    E.spmm_csr_rows(*csr, dr, dX, None, acc=a2, acc_scale=-1.5)
    assert torch.equal(a1, a2)
    np.testing.assert_allclose(a1.cpu().numpy()[rows], acc0[rows] - 1.5 * ref[rows], rtol=1e-4, atol=4e-6)
    # empty list
    E.spmm_csr_rows(*csr, torch.zeros(0, dtype=torch.int32, device='cuda'), dX, Y)


@pytest.mark.parametrize('d,world,n', [(64, 8, 2048), (64, 2, 777), (128, 4, 5000), (16, 4, 33), (256, 2, 100)])
def test_bpr_column_block_step_equals_fused_kernel(torch, E, d, world, n):
    """Feature-parallel K3: partial scores per column block, summed (the all-reduce), then the gradient of each block
    from the full scores -- together the fused kernel's gradient and loss (the -ln terms counted once, the L2 term in
    column parts), for every block width down to 8 columns."""
    rng = np.random.default_rng(d + world + n)
    nu, ni = 300, 170
    U = (rng.standard_normal((nu, d)) * 0.2).astype(np.float32)
    V = (rng.standard_normal((ni, d)) * 0.2).astype(np.float32)
    u, i, j = (rng.integers(0, hi, n).astype(np.int32) for hi in (nu, ni, ni))
    du, di, dj = _dev(torch, u), _dev(torch, i), _dev(torch, j)
    gU, gV = torch.zeros(nu, d, device='cuda'), torch.zeros(ni, d, device='cuda')
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    E.bpr_grad_scatter(_dev(torch, U), _dev(torch, V), du, di, dj, 10e-8, 0.001, gU, gV, loss)
    dw = d // world
    blocks = [(_dev(torch, np.ascontiguousarray(U[:, r * dw:(r + 1) * dw])), _dev(torch, np.ascontiguousarray(V[:, r * dw:(r + 1) * dw])))
              for r in range(world)]
    losses = torch.zeros(world, dtype=torch.float64, device='cuda')
    parts = torch.full((world, n), 7.0, device='cuda')
    for r, (Ub, Vb) in enumerate(blocks):
        E.bpr_partial_scores(Ub, Vb, du, di, dj, 0.001, parts[r], losses[r:r + 1])
    y = parts.sum(0).contiguous()
    ref_y = (U[u].astype(np.float64) * (V[i].astype(np.float64) - V[j].astype(np.float64))).sum(1)
    np.testing.assert_allclose(y.cpu().numpy(), ref_y, rtol=1e-4, atol=1e-6)
    got_U, got_V = torch.zeros(nu, d, device='cuda'), torch.zeros(ni, d, device='cuda')
    for r, (Ub, Vb) in enumerate(blocks):
        gu, gv = torch.zeros(nu, dw, device='cuda'), torch.zeros(ni, dw, device='cuda')
        E.bpr_grad_from_scores(Ub, Vb, du, di, dj, y, 10e-8, 0.001, 1.0 if r == 0 else 0.0, gu, gv, losses[r:r + 1])
        got_U[:, r * dw:(r + 1) * dw] = gu
        got_V[:, r * dw:(r + 1) * dw] = gv
    torch.testing.assert_close(got_U, gU, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(got_V, gV, rtol=1e-4, atol=1e-6)
    assert abs(losses.sum().item() - loss.item()) <= 1e-6 * abs(loss.item())
