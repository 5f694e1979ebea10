"""K8 (csrc/topn_kernels.cu): fused score + rated-mask + top-N against the reference's per-user flow
(base/recommender.py:143-152 + util/qmath.py:134-146) restated in numpy: candidates = Q.dot(P[u]),
rated items := 0, N best by (score desc, item id asc).  Index lists must be EXACT wherever the fp32 scores
are distinct; scores equal to the numpy dot to fp32 rounding."""
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


def _reference(P, Q, users, rp, co, N, rated_value=0.0):
    ids, vals = [], []
    for u in users:
        s = (Q.astype(np.float64) @ P[u].astype(np.float64)).astype(np.float32)
        s[co[rp[u]:rp[u + 1]]] = rated_value
        top = np.lexsort((np.arange(len(s)), -s))[:N]
        ids.append(top); vals.append(s[top])
    return np.array(ids), np.array(vals)


def _csr(rng, nu, ni, max_deg):
    deg = rng.integers(0, max_deg + 1, nu)
    rp = np.zeros(nu + 1, np.int64); rp[1:] = np.cumsum(deg)
    co = np.concatenate([np.sort(rng.choice(ni, k, replace=False)) for k in deg] + [np.zeros(0, np.int64)]).astype(np.int32)
    return rp, co


@pytest.mark.parametrize('nu,ni,d,N,signed,tc', [(130, 1000, 64, 10, False, False), (77, 333, 52, 100, True, False), (5, 150, 8, 50, True, False),
                                                 (300, 20000, 64, 20, False, False), (64, 129, 128, 100, True, False),
                                                 # the wgmma 3xTF32 kernel (d <= 64): same bounds -- fp32-level scores
                                                 (130, 1000, 64, 10, False, True), (77, 333, 32, 100, True, True), (5, 150, 64, 50, True, True),
                                                 (300, 20000, 64, 20, False, True), (129, 257, 32, 100, True, True), (90, 700, 52, 30, True, True), (40, 300, 8, 20, False, True),
                                                 (1000, 5000, 64, 100, True, True)])
def test_topn_equals_reference_flow(torch, E, nu, ni, d, N, signed, tc):
    rng = np.random.default_rng(nu * 7 + ni)
    P = (rng.standard_normal((nu, d)) if signed else rng.random((nu, d))).astype(np.float32)
    Q = (rng.standard_normal((ni, d)) if signed else rng.random((ni, d))).astype(np.float32)
    rp, co = _csr(rng, nu, ni, min(60, ni // 2))
    users = rng.permutation(nu)[:max(1, nu - 3)].astype(np.int32)
    ids, vals = E.score_topn(torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda(), torch.from_numpy(users).cuda(),
                             torch.from_numpy(rp).cuda(), torch.from_numpy(co).cuda(), N, tensor_cores=tc)
    torch.cuda.synchronize()
    ids, vals = ids.cpu().numpy(), vals.cpu().numpy()
    rid, rval = _reference(P, Q, users, rp, co, N)
    assert np.all(np.diff(vals, axis=1) <= 0)
    np.testing.assert_allclose(vals, rval, rtol=2e-5, atol=2e-5)
    # exact index parity wherever the reference scores are separated by more than fp32 summation noise
    for r in range(len(users)):
        gap_ok = np.ones(N, bool)
        gap_ok[1:] &= (rval[r, :-1] - rval[r, 1:]) > 1e-4
        gap_ok[:-1] &= (rval[r, :-1] - rval[r, 1:]) > 1e-4
        assert np.array_equal(ids[r][gap_ok], rid[r][gap_ok]), 'row %d' % r
        # rated items that made the list carry exactly the rated value
        rated = set(co[rp[users[r]]:rp[users[r] + 1]].tolist())
        assert all((k not in rated) or v == 0.0 for k, v in zip(ids[r].tolist(), vals[r].tolist()))
        assert len(set(ids[r].tolist())) == N


@pytest.mark.parametrize('tc', [False, True])
def test_topn_ties_and_rated_zeros_outrank_negative_scores(torch, E, tc):
    """All unrated scores negative, so the rated items (score 0) must fill the top of the list (the reference
    writes 0, it does not remove them -- SURVEY A7); exact ties are ordered by ascending item id."""
    nu, ni, d, N = 3, 400, (32 if tc else 4), 12
    P = np.zeros((nu, d), np.float32); P[:, :4] = 1.0
    Q = np.zeros((ni, d), np.float32); Q[:, :4] = -1.0     # every raw score is exactly -4
    Q[100:110, :4] = -0.5                                   # ten items score exactly -2 (a tie block)
    rp = np.array([0, 5, 5, 9], np.int64)
    co = np.array([3, 50, 150, 250, 399, 0, 1, 2, 398], np.int32)
    ids, vals = E.score_topn(torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda(), torch.arange(3, dtype=torch.int32).cuda(),
                             torch.from_numpy(rp).cuda(), torch.from_numpy(co).cuda(), N, tensor_cores=tc)
    ids, vals = ids.cpu().numpy(), vals.cpu().numpy()
    assert ids[0].tolist() == [3, 50, 150, 250, 399] + list(range(100, 107))
    assert vals[0].tolist() == [0.0] * 5 + [-2.0] * 7
    assert ids[1].tolist() == list(range(100, 110)) + [0, 1] and vals[1].tolist() == [-2.0] * 10 + [-4.0] * 2
    assert ids[2].tolist() == [0, 1, 2, 398] + list(range(100, 108))


def test_topn_bad_arguments(torch, E):
    U = torch.ones(4, 8, device='cuda'); V = torch.ones(5, 8, device='cuda')
    rp = torch.zeros(5, dtype=torch.int64, device='cuda'); co = torch.zeros(1, dtype=torch.int32, device='cuda')
    u = torch.arange(4, dtype=torch.int32, device='cuda')
    with pytest.raises(E.QRecError):
        E.score_topn(U, V, u, rp, co, 6)                   # N > items
    with pytest.raises(E.QRecError):
        E.score_topn(torch.ones(4, 8, device='cuda'), torch.ones(200, 8, device='cuda'), u, rp, co, 102)   # N > 101
    with pytest.raises(E.QRecError):
        E.score_topn(torch.ones(4, 8, device='cuda'), torch.ones(200, 8, device='cuda'), u, rp, co, 102, tensor_cores=False)
    ids, _ = E.score_topn(U, V, u[:0], rp, co, 3)          # empty block
    assert ids.shape == (0, 3)
    with pytest.raises(E.QRecError):
        E.score_topn(torch.ones(4, 128, device='cuda'), torch.ones(5, 128, device='cuda'), u, rp, co, 3, tensor_cores=True)   # d > 64


def test_topn_tensor_core_kernel_agrees_with_simt_kernel(torch, E):
    """Both kernels on one larger block (2048 users x 30000 items, d = 64, N = 100): identical index lists wherever the
    SIMT scores are separated by more than fp32 summation noise, scores within 2e-5."""
    g = torch.Generator(device='cuda'); g.manual_seed(5)
    nu, ni, d, N = 2048, 30000, 64, 100
    P = torch.randn(nu, d, device='cuda', generator=g); Q = torch.randn(ni, d, device='cuda', generator=g)
    rng = np.random.default_rng(5)
    rp, co = _csr(rng, nu, ni, 40)
    users = torch.arange(nu, dtype=torch.int32, device='cuda')
    a_ids, a_val = E.score_topn(P, Q, users, torch.from_numpy(rp).cuda(), torch.from_numpy(co).cuda(), N, tensor_cores=False)
    b_ids, b_val = E.score_topn(P, Q, users, torch.from_numpy(rp).cuda(), torch.from_numpy(co).cuda(), N, tensor_cores=True)
    torch.cuda.synchronize()
    a_ids, a_val, b_ids, b_val = (x.cpu().numpy() for x in (a_ids, a_val, b_ids, b_val))
    np.testing.assert_allclose(b_val, a_val, rtol=2e-5, atol=2e-5)
    gap = np.ones_like(a_val, bool)
    sep = (a_val[:, :-1] - a_val[:, 1:]) > 1e-4
    gap[:, 1:] &= sep; gap[:, :-1] &= sep
    assert np.array_equal(a_ids[gap], b_ids[gap]) and gap.mean() > 0.9
