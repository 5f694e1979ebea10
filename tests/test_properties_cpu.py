"""Property tests (hypothesis) of the host-side building blocks: the structures the kernels index into
must agree with the reference's dict-of-dicts semantics for ANY interaction list."""
import random

import numpy as np
import torch
from hypothesis import given, settings, strategies as st

from qrec_b200 import engine as E
from qrec_b200 import parallel
from qrec_b200.data.interactions import InteractionTable

records = st.lists(st.tuples(st.integers(0, 12), st.integers(0, 15), st.sampled_from([0.5, 1.0, 2.0, 4.0])),
                   min_size=0, max_size=120)


@settings(max_examples=150, deadline=None)
@given(records)
def test_rated_csr_is_the_dict_of_dicts(recs):
    nu, ni = 13, 16
    u = np.array([r[0] for r in recs], dtype=np.int64)
    i = np.array([r[1] for r in recs], dtype=np.int64)
    r = np.array([r[2] for r in recs], dtype=np.float64)
    csr = E.RatedCSR(nu, ni, u, i, r)
    rows = [dict() for _ in range(nu)]
    for a, b, c in recs:
        rows[a][b] = c                          # insertion position of the first write, value of the last
    for a in range(nu):
        s0, s1 = csr.sorted_rowptr[a], csr.sorted_rowptr[a + 1]
        assert csr.sorted_cols[s0:s1].tolist() == sorted(rows[a])
        p0, p1 = csr.pos_rowptr[a], csr.pos_rowptr[a + 1]
        assert csr.pos_cols[p0:p1].tolist() == [k for k, v in rows[a].items() if v >= 1]
        assert csr.possorted_cols[p0:p1].tolist() == sorted(k for k, v in rows[a].items() if v >= 1)


@settings(max_examples=100, deadline=None)
@given(st.lists(st.sampled_from(['a', 'b', 'c', 'dd', 'e1', 'zz', '7', '10']), min_size=0, max_size=60))
def test_first_appearance_ids(names):
    ids, vocab = (InteractionTable._first_appearance_ids(np.array(names)) if names
                  else (np.zeros(0, np.int32), np.zeros(0, str)))
    d = {}
    for n in names:
        if n not in d:
            d[n] = len(d)
    assert ids.tolist() == [d[n] for n in names] and vocab.tolist() == list(d)


@settings(max_examples=60, deadline=None)
@given(st.integers(0, 2**40), st.integers(0, 400))
def test_mt_clone_shuffle_and_randbelow_track_cpython(seed, n):
    r = random.Random(seed)
    m = E.MT19937(seed)
    x = list(range(n))
    r.shuffle(x)
    a = np.arange(n, dtype=np.int32)
    m.shuffle(a)
    assert a.tolist() == x
    for bound in (1, 2, 3, 1000, 2**31 - 1):
        assert m.randbelow(bound) == r._randbelow(bound)
    assert m.random() == r.random() and m.getstate() == r.getstate()


@settings(max_examples=60, deadline=None)
@given(st.integers(1, 8), st.integers(1, 40), st.integers(1, 30))
def test_node_partition_is_a_bijection(world, bu, bi):
    U, I = world * bu, world * bi
    part = parallel.NodePartition(U, I, world)
    g = part.to_gathered(torch.arange(U + I))
    assert sorted(g.tolist()) == list(range(U + I))
    seen = torch.cat([part.local_nodes(r) for r in range(world)])
    assert sorted(seen.tolist()) == list(range(U + I))
    for r in range(world):                       # a rank's nodes occupy exactly its block of the gathered order
        pos = part.to_gathered(part.local_nodes(r))
        assert pos.tolist() == list(range(r * part.block, (r + 1) * part.block))


@settings(max_examples=80, deadline=None)
@given(records, st.integers(1, 4))
def test_bipartite_shards_tile_the_adjacency(recs, world):
    """shard_bipartite_by_user: the ranks' A_ui blocks stack to the user rows of the joint matrix and each
    A_iu block is the transpose of its A_ui block."""
    from oracle import bpr_oracle as O
    nu, ni = 13, 16
    if not recs:
        return
    u = np.array([r[0] for r in recs]); i = np.array([r[1] for r in recs])
    A = O.norm_adjacency(nu, ni, u, i)
    rp, co, va = (torch.from_numpy(x) for x in (A.indptr.astype(np.int64), A.indices.astype(np.int32), A.data))
    dense = A.toarray()
    for rank in range(world):
        A_ui, A_iu, (lo, hi) = parallel.shard_bipartite_by_user(rp, co, va, nu, ni, rank, world)
        if hi == lo:
            continue
        D_ui = torch.sparse_csr_tensor(A_ui[0], A_ui[1].long(), A_ui[2], size=(hi - lo, ni)).to_dense().numpy()
        D_iu = torch.sparse_csr_tensor(A_iu[0], A_iu[1].long(), A_iu[2], size=(ni, hi - lo)).to_dense().numpy()
        assert np.array_equal(D_ui, dense[lo:hi, nu:]) and np.array_equal(D_iu, D_ui.T)


@settings(max_examples=120, deadline=None)
@given(records)
def test_row_version_schedule_replays_the_sequential_order(recs):
    """qrec_mf_order_prepare / qrec_bpr_order_prepare: executing entries whenever their rows have reached
    the recorded versions (any admissible interleaving, here: always the LAST ready entry) touches every
    row in exactly the sequential order, and the depth is the longest dependency chain."""
    nu, ni = 13, 16
    u = np.array([r[0] for r in recs], dtype=np.int32)
    i = np.array([r[1] for r in recs], dtype=np.int32)
    wu, wi = E.mf_order_prepare(u, i, nu, ni)
    ver_p, ver_q = np.zeros(nu, int), np.zeros(ni, int)
    pending = list(range(len(recs)))
    seen_p, seen_q = [[] for _ in range(nu)], [[] for _ in range(ni)]
    while pending:
        ready = [k for k in pending if ver_p[u[k]] == wu[k] and ver_q[i[k]] == wi[k]]
        assert ready and pending[0] in ready            # the oldest entry is always runnable: no deadlock
        k = ready[-1]
        pending.remove(k)
        seen_p[u[k]].append(k); seen_q[i[k]].append(k)
        ver_p[u[k]] += 1; ver_q[i[k]] += 1
    for a in range(nu):
        assert seen_p[a] == [k for k in range(len(recs)) if u[k] == a]
    for b in range(ni):
        assert seen_q[b] == [k for k in range(len(recs)) if i[k] == b]
    level_p, level_q, depth = np.zeros(nu, int), np.zeros(ni, int), 0
    for k in range(len(recs)):
        lv = max(level_p[u[k]], level_q[i[k]]) + 1
        level_p[u[k]] = level_q[i[k]] = lv
        depth = max(depth, lv)
    assert E.mf_order_depth(u, i, nu, ni) == depth
    # the pairwise version with j = (i + 1) mod ni shares the item counters between both item rows
    j = ((i + 1) % ni).astype(np.int32)
    bu, bi, bj = E.bpr_order_prepare(u, i, j, nu, ni)
    cq = np.zeros(ni, int)
    for k in range(len(recs)):
        assert bu[k] == wu[k] and bi[k] == cq[i[k]] and bj[k] == cq[j[k]]          # i != j here
        cq[i[k]] += 1; cq[j[k]] += 1


@settings(max_examples=80, deadline=None)
@given(records, st.integers(1, 5))
def test_column_blocks_sum_to_the_matrix(recs, n_blocks):
    """parallel.split_csr_columns: the blocks partition the non-zeros by column range, keep every row's
    order, and blocked_spmm over them equals the unsplit product."""
    import scipy.sparse as sp
    nu, ni = 13, 16
    M = sp.csr_matrix((np.array([r[2] for r in recs], np.float32),
                       (np.array([r[0] for r in recs], int), np.array([r[1] for r in recs], int))), shape=(nu, ni))
    M.sum_duplicates(); M.sort_indices()
    csr = (torch.from_numpy(M.indptr.astype(np.int64)), torch.from_numpy(M.indices.astype(np.int32)),
           torch.from_numpy(M.data.astype(np.float32)))
    blocks = parallel.split_csr_columns(csr, ni, n_blocks)
    assert len(blocks) == max(1, n_blocks)
    width = -(-ni // n_blocks)
    total = np.zeros((nu, ni), np.float32)
    for b, (rp, co, va) in enumerate(blocks):
        assert rp.dtype == torch.int64 and co.dtype == torch.int32 and int(rp[-1]) == co.numel() == va.numel()
        if n_blocks > 1:
            assert bool(((co >= b * width) & (co < (b + 1) * width)).all())
        D = sp.csr_matrix((va.numpy(), co.numpy(), rp.numpy()), shape=(nu, ni))
        assert D.has_sorted_indices or D.nnz == 0
        total += D.toarray()
    assert np.array_equal(total, M.toarray())

    def spmm(A, X, Y, acc, s):
        D = torch.from_numpy(sp.csr_matrix((A[2].numpy(), A[1].numpy(), A[0].numpy()), shape=(nu, ni)).toarray())
        Y.copy_(D @ X)
        if acc is not None:
            acc.add_(Y, alpha=s)
    X = torch.arange(ni * 3, dtype=torch.float32).reshape(ni, 3) / 7
    Y, scratch, acc = torch.full((nu, 3), 9.0), torch.full((nu, 3), 5.0), torch.ones(nu, 3)
    parallel.blocked_spmm(spmm, blocks, X, Y, scratch, acc, 0.5)
    ref = torch.from_numpy(M.toarray()) @ X
    assert torch.allclose(Y, ref, atol=1e-5) and torch.allclose(acc, 1 + 0.5 * ref, atol=1e-5)


@settings(max_examples=150, deadline=None)
@given(records, st.sampled_from([0.5, 1.0, 2.5]))
def test_native_rated_csr_equals_numpy_construction(recs, threshold):
    """qrec_build_rated_csr (counting sort + per-user sorts, threaded) against the numpy construction it
    replaced (oracle.rated_csr_numpy): all five arrays, for repeated pairs, empty users and mixed ratings."""
    from oracle import bpr_oracle as O
    nu, ni = 13, 16
    u = np.array([r[0] for r in recs], dtype=np.int64)
    i = np.array([r[1] for r in recs], dtype=np.int64)
    r = np.array([r[2] for r in recs], dtype=np.float64)
    got = E.RatedCSR(nu, ni, u, i, r, positive_threshold=threshold)
    want = O.rated_csr_numpy(nu, ni, u, i, r, positive_threshold=threshold)
    assert np.array_equal(got.sorted_rowptr, want['sorted_rowptr']) and np.array_equal(got.sorted_cols, want['sorted_cols'])
    assert np.array_equal(got.pos_rowptr, want['pos_rowptr']) and np.array_equal(got.pos_cols, want['pos_cols'])
    assert np.array_equal(got.possorted_rowptr, got.pos_rowptr if len(got.pos_cols) != len(got.sorted_cols) else got.sorted_rowptr)
    assert np.array_equal(got.possorted_cols, want['possorted_cols'])


def test_native_rated_csr_large_threaded_and_errors():
    from oracle import bpr_oracle as O
    rng = np.random.default_rng(3)
    nu, ni, n = 40000, 5000, 1_500_000                    # several threads, repeated pairs, skewed users
    u = np.minimum(rng.zipf(1.3, n) - 1, nu - 1).astype(np.int64)
    i = rng.integers(0, ni, n)
    r = rng.integers(0, 5, n) / 1.0
    got = E.RatedCSR(nu, ni, u, i, r)
    want = O.rated_csr_numpy(nu, ni, u, i, r)
    for k in ('sorted_rowptr', 'sorted_cols', 'pos_rowptr', 'pos_cols', 'possorted_cols'):
        assert np.array_equal(getattr(got, k), want[k]), k
    import pytest
    with pytest.raises(E.QRecError):
        E.RatedCSR(3, 4, np.array([0, 3]), np.array([1, 1]))          # user id out of range
    with pytest.raises(E.QRecError):
        E.RatedCSR(3, 4, np.array([0, 1]), np.array([1, -1]))         # negative item id
    with pytest.raises(E.QRecError):
        E.RatedCSR(3, 4, np.array([0, 1]), np.array([1]))


def test_device_csr_split_row_issues_one_launch_per_half_with_the_same_result(monkeypatch):
    """DeviceCSR.set_split_row: matmul over the joint adjacency = the row-split product over rows [0, split) and over
    rows [split, n), each a row range of the same CSR (rowptr slice with absolute offsets into cols / vals)."""
    import scipy.sparse as sp
    import torch
    from qrec_b200 import engine as E
    from qrec_b200.base.graphRecommender import DeviceCSR
    rng = np.random.default_rng(4)
    nu, ni, d = 23, 9, 8
    R = (rng.random((nu, ni)) < 0.3).astype(np.float32)
    A = sp.bmat([[None, sp.csr_matrix(R)], [sp.csr_matrix(R.T), None]], format='csr').astype(np.float32)
    A.data[:] = rng.random(A.nnz).astype(np.float32)
    calls = []

    def spmm(rowptr, cols, vals, X, Y, acc=None, acc_scale=0.0, rowsplit=False):
        rp = rowptr.numpy()
        a, b = int(rp[0]), int(rp[-1])
        calls.append((rowptr.numel() - 1, a, b, rowsplit))
        M = sp.csr_matrix((vals.numpy()[a:b], cols.numpy()[a:b], rp - a), shape=(rowptr.numel() - 1, X.shape[0]))
        Y.copy_(torch.from_numpy(M @ X.numpy()))
        if acc is not None:
            acc.add_(Y, alpha=acc_scale)
        return Y
    monkeypatch.setattr(E, 'spmm_csr', spmm)
    X = torch.from_numpy(rng.standard_normal((nu + ni, d)).astype(np.float32))
    ref = torch.from_numpy(A @ X.numpy())
    whole = DeviceCSR(A, 'cpu')
    assert whole.split_row is None
    Y0, acc0 = torch.empty_like(X), torch.ones_like(X)
    whole.matmul(X, Y0, acc=acc0, acc_scale=0.5)
    assert len(calls) == 1 and calls[0][0] == nu + ni
    split = DeviceCSR.from_tensors(A.shape, whole.rowptr, whole.cols, whole.vals, split_row=nu)
    assert split.split_row == nu
    calls.clear()
    Y1, acc1 = torch.full_like(X, 7.0), torch.ones_like(X)
    split.matmul(X, Y1, acc=acc1, acc_scale=0.5)
    nnz_u = int(whole.rowptr[nu])
    assert calls == [(nu, 0, nnz_u, True), (ni, nnz_u, A.nnz, True)]
    assert torch.allclose(Y0, ref, atol=1e-6) and torch.equal(Y1, Y0) and torch.equal(acc1, acc0)
    # out-of-range split rows leave the single launch
    assert DeviceCSR.from_tensors(A.shape, whole.rowptr, whole.cols, whole.vals, split_row=0).split_row is None
    assert DeviceCSR.from_tensors(A.shape, whole.rowptr, whole.cols, whole.vals, split_row=nu + ni).split_row is None
