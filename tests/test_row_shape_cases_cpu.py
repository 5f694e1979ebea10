"""The cases of test_gpu_row_shape_matrix.py checked without a GPU: the width tables reach every lane-group shape each
launcher is compiled for, with all lanes busy and with idle lanes (through the host build of lane_shape.h); the
builders reach every branch they are named for; and the references that are new in row_shape_cases.py agree with the
existing oracles."""
import numpy as np
import pytest

import row_shape_cases as R
from test_lane_shape_cpu import lib, shape  # noqa: F401

ROW_LAUNCHERS = [k for k, cap in R.LAUNCHERS.items() if cap != 'parity']


def host_shape(lib, d, cap):  # noqa: F811
    lpr, vpl, _ = shape(lib, d // 4, cap)
    return lpr, vpl


def test_row_shape_restatement_is_the_dispatch(lib):  # noqa: F811
    for cap in (128, 256):
        for d in range(4, cap + 1, 4):
            assert R.row_shape(d, cap) == host_shape(lib, d, cap)
    assert all(R.lane_elems(d) == lib.lane_elems_host(d) for d in range(1, 257))


@pytest.mark.parametrize('launcher', list(R.LAUNCHERS))
def test_widths_reach_every_shape_busy_and_idle(lib, launcher):  # noqa: F811
    """(LPR, VPL) of the row kernels and E of the parity kernels, each with d filling every lane and with idle lanes."""
    cap = R.LAUNCHERS[launcher]
    if cap == 'parity':
        reached = {(lib.lane_elems_host(d), d == 32 * lib.lane_elems_host(d)) for d in R.widths(launcher)}
        assert reached == {(e, busy) for e in (1, 2, 4, 8) for busy in (True, False)}
        return
    reached = set()
    for d in R.widths(launcher):
        if launcher == 'spmm_rowsplit' and d == 64:
            continue                               # spmm_csr_d64_kernel, not the template
        lpr, vpl = host_shape(lib, d, cap)
        reached.add((lpr, vpl, d == 4 * lpr * vpl))
    shapes = [(4, 1), (8, 1), (16, 1), (32, 1)] + ([(32, 2)] if cap == 256 else [])
    expected = {(lpr, vpl, busy) for lpr, vpl in shapes for busy in (True, False)}
    if launcher == 'spmm_rowsplit':
        # nvec = 16 is d = 64 only, which the row-split launcher hands to its d = 64 kernel: the template at (16, 1)
        # runs with idle lanes alone
        expected.discard((16, 1, True))
        assert 64 in R.widths(launcher)
    assert reached == expected
    assert max(R.widths(launcher)) == cap


@pytest.mark.parametrize('launcher', [k for k in ROW_LAUNCHERS if k.startswith('spmm')])
def test_spmm_tails_reach_every_row_length_tail(launcher):
    for d in R.widths(launcher):
        lpr, vpl = R.row_shape(d, R.LAUNCHERS[launcher])
        c = R.spmm_case(launcher, d, 'tails')
        lengths = set(np.diff(c['rowptr']).tolist())
        gather = {'spmm_balanced': 4, 'spmm_rowsplit': R.rowsplit_gather(vpl), 'spmm_rows': 4 * 32 // lpr,
                  'spmm_scatter_rows': R.SLICE}[launcher]
        need = {0, 1, lpr - 1, lpr, lpr + 1, 2 * lpr + 1}
        need |= set(range(0, 2 * lpr + 2, lpr)) | set(range(0, 2 * lpr + 2, min(gather, 2 * lpr + 1)))
        need |= {gather - 1, gather, gather + 1, 2 * gather - 1, 2 * gather, 2 * gather + 1}
        assert need <= lengths, sorted(need - lengths)
        assert np.diff(c['rowptr'])[[0, -1]].tolist() == [0, 0]
        if c['rows'] is not None:
            assert (c['rows'] == -1).any()
            listed = c['rows'][c['rows'] >= 0]
            assert np.all(np.diff(listed) > 0)
        if launcher == 'spmm_scatter_rows':
            # more (source row, slice) work items than the launch has lane groups: every group takes grid-stride rounds
            assert len(c['rows']) * R.PASS > R.lane_groups(lpr)


@pytest.mark.parametrize('launcher', [k for k in ROW_LAUNCHERS if k.startswith('spmm')])
def test_spmm_long_rows(launcher):
    for d in R.widths(launcher):
        c = R.spmm_case(launcher, d, 'long')
        rp = c['rowptr']
        deg = np.diff(rp)
        listed = np.arange(len(deg)) if c['rows'] is None else c['rows'][c['rows'] >= 0]
        long_rows = listed[deg[listed] > R.CHUNK]
        assert len(long_rows) >= 5
        # rows longer than one pass of the scatter kernel (64 slices of 64 edges) take a second and a third pass
        assert deg[listed].max() > 2 * R.SLICE * R.PASS and (deg[listed] == R.SLICE * R.PASS + 1).any()
        # rows that straddle a balanced chunk boundary, and long rows with empty rows after them
        straddle = (rp[:-1] // R.CHUNK) != ((rp[1:] - 1) // R.CHUNK)
        assert (straddle & (deg > 0) & (deg < R.CHUNK)).any() and (straddle & (deg > R.CHUNK)).any()
        assert all(deg[r + 1] == 0 for r in np.nonzero(deg > R.CHUNK)[0])
        if c['rows'] is not None:
            assert (c['rows'] == -1).any()


def test_spmm_defect_drops_one_entry_per_row():
    c = R.spmm_case('spmm_balanced', 20, 'tails')
    A, B = R.csr_matrix(c), R.csr_matrix(c, drop_last=True)
    deg = np.diff(c['rowptr'])
    assert A.nnz - B.nnz == (deg > 0).sum()
    assert np.array_equal(np.diff(B.indptr), np.maximum(deg - 1, 0))


@pytest.mark.parametrize('structure', list(R.K3_SIZES))
def test_k3_batches(structure):
    for d in R.widths('k3'):
        c = R.k3_case(d, structure)
        u, i, j = c['u'], c['i'], c['j']
        ok = u >= 0
        assert (~ok).any() and ok.sum() >= 3 and len(u) % 32 != 0
        # conflict-free: no gradient row is scattered to twice
        assert len(np.unique(u[ok])) == ok.sum() and len(np.unique(np.concatenate([i, j]))) == 2 * len(u)
        assert len(c['gU0']) > ok.sum() and len(c['gV0']) > 2 * len(u)
    assert R.K3_SIZES['short'] < 8 < R.K3_SIZES['batch']     # fewer triples than one lane group's first step, and many


def test_k3_reference_is_bpr_loss_grad():
    from oracle import bpr_oracle as O
    c = R.k3_case(36, 'batch')
    ok = c['u'] >= 0
    args = c['U'], c['V'], c['u'], c['i'], c['j'], 1e-7, 0.01
    loss, gU, gV, _ = R.k3_reference(*args, 'grad')
    rl, rU, rV = O.bpr_loss_grad(c['U'], c['V'], c['u'][ok], c['i'][ok], c['j'][ok], 1e-7, 0.01)
    assert abs(loss - rl) <= 1e-12 * abs(rl)
    np.testing.assert_allclose(gU, rU, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(gV, rV, rtol=1e-12, atol=1e-15)
    # unit scales are the plain entry; the full scores of the tables give its gradients and its -ln terms
    ones = np.ones(len(c['u']), np.float32)
    s = R.k3_reference(*args, 'scaled', y_scale=ones)
    assert s[0] == loss and np.array_equal(s[1], gU) and np.array_equal(s[2], gV)
    l2, _, _, y = R.k3_reference(*args, 'partial_scores')
    assert np.all(y[~ok] == 0)
    f = R.k3_reference(*args, 'grad_from_scores', y_full=y, log_weight=1.0)
    assert abs(f[0] + l2 - loss) <= 1e-12 * abs(loss)
    np.testing.assert_allclose(f[1], gU, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize('structure', ['ragged', 'grid_stride'])
def test_staged_batches(structure):
    for d in R.widths('bpr_staged'):
        c = R.staged_case(d, structure)
        n, lpr = len(c['u']), R.row_shape(d, 128)[0]
        assert len(np.unique(c['u'])) == n and len(np.unique(np.concatenate([c['pos_i'], c['pos_j']]))) == 2 * n
        assert len(c['R']) > 2 * n and len(c['P']) > n
        if structure == 'grid_stride':
            assert n > R.staged_groups(lpr) and n % R.staged_groups(lpr) != 0
        else:
            assert n < R.staged_groups(lpr) and n % 32 != 0


def test_staged_reference_is_the_bpr_step():
    """On staged rows the step is BPR.py:45-53 as bpr_sgd_jacobi states it, with Q[i] = R[pos_i], Q[j] = R[pos_j]."""
    from oracle import bpr_oracle as O
    c = R.staged_case(20, 'ragged')
    u, pi, pj = c['u'][:300], c['pos_i'][:300], c['pos_j'][:300]
    P, D, loss = R.staged_reference(c['P'], c['R'], c['D0'], u, pi, pj, 0.05, 0.01, 0.02)
    dP, dQ, rl = O.bpr_sgd_jacobi(c['P'], c['R'], list(zip(u, pi, pj)), 0.05, 0.01, 0.02)
    np.testing.assert_allclose(P, c['P'] + dP, rtol=1e-12, atol=1e-15)
    w = np.concatenate([pi, pj])
    np.testing.assert_allclose(D[w], dQ[w], rtol=1e-12, atol=1e-15)
    assert abs(loss - rl) <= 1e-12 * rl
    keep = np.ones(len(D), bool)
    keep[w] = False
    assert np.array_equal(D[keep], c['D0'][keep])


@pytest.mark.parametrize('structure', ['ragged', 'windowed'])
def test_mf_batches(structure):
    for d in R.widths('mf_batch'):
        c = R.mf_batch_case(d, structure)
        n = len(c['u'])
        assert len(np.unique(c['u'])) == n and len(np.unique(c['i'])) == n
        assert len(c['P']) > n and len(c['Q']) > n and not c['P'][:, d - R.PAD:].any()
        if structure == 'windowed':
            # more entries than the bounded launch holds in flight (4 per lane group): grid-stride rounds
            assert n > 4 * R.mf_batch_groups(d, c['max_inflight'])
        else:
            assert c['max_inflight'] == 0 and n % 32 != 0


def test_mf_ordered_entries_repeat_rows():
    for dt in (np.float32, np.float64):
        c = R.mf_ordered_case(64, dt)
        assert c['P'].dtype == dt and c['r'].dtype == dt
        assert np.bincount(c['u']).min() > 5 and np.bincount(c['i']).min() > 5


@pytest.mark.parametrize('structure', ['one_in_flight', 'disjoint'])
def test_svdpp_users(structure):
    for d in R.widths('svdpp_usermajor'):
        c = R.svdpp_case(d, structure)
        W = np.diff(c['rowptr'])[c['order']]
        empty = np.nonzero(W == 0)[0]
        assert len(empty) and empty.min() > 0 and empty.max() < len(W) - 1, 'W = 0 users inside the row order'
        assert {w % R.K_PREFETCH for w in W[W > 0]} == {0, 1, 2, 3} and (W == 1).any()
        assert (W > 4 * R.K_PREFETCH).any()
        for t in c['tabs'][:3]:
            assert not t[:, d - R.PAD:].any()
        rated = np.unique(c['cols'])
        assert len(rated) < len(c['tabs'][1])                  # items no user rated: rows the epoch must not touch
        users = (W > 0).sum()
        if structure == 'disjoint':
            assert len(rated) == len(c['cols'])
            assert 1 < c['in_flight'] < users
        else:
            assert c['in_flight'] == 1 and len(rated) < len(c['cols'])


def test_defects_move_what_they_claim():
    tabs = [np.ones((3, 12), np.float32), np.ones(3, np.float32)]
    z = R.zero_last_slice(tabs, 12)
    assert not z[0][:, 8:].any() and z[0][:, :8].all() and z[1].all() and tabs[0].all()
    assert R.sum_ratio(np.array([1.0, 0.0]), np.array([1.0, 0.0]), np.array([1.0, 0.0])) == 0.0
    assert R.sum_ratio(np.array([1.0, 1e-30]), np.array([1.0, 0.0]), np.array([1.0, 0.0])) == float('inf')
