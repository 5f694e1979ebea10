"""The K8 top-N cases (topn_cases.py) without a GPU: their scores are exact under every way the two kernels sum them,
they reach every compaction, tail and signature branch of both kernels, every defect reference is told apart by the
families that target it, and `evaluate.batched_top_n` -- the `-eval gpu` ranking -- returns the reference heap's lists
when the kernel it drives keeps the kernel contract."""
import numpy as np
import pytest

import topn_cases as T


def _tables(case):
    return case.U, case.V, np.unique(case.users)


@pytest.mark.parametrize('case', T.CASES, ids=repr)
def test_scores_are_exact_in_fp32_fma_and_tf32(case):
    U, V, users = _tables(case)
    assert np.all(U == np.round(U)) and np.all(V == np.round(V))
    assert np.abs(U).max() <= 8 and np.abs(V).max() <= 8 and case.d <= 256
    s64 = T.scores64(U, V, users)
    fma, peak = T.fma_scores_f32(U, V, users)
    assert np.array_equal(fma.astype(np.float64), s64)
    assert peak <= 2.0 ** 14 < 2.0 ** 24                    # every partial sum is an exact fp32 integer
    for X in (U, V):                                         # the 3xTF32 operands: hi = x, lo = 0
        hi, lo = T.tf32_split(X)
        assert np.array_equal(hi, X) and not np.any(lo)


def test_tf32_emulation_rounds_to_nearest_away():
    x = np.array([1.0 + 2.0 ** -11, 1.0 + 2.0 ** -10 + 2.0 ** -11, -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -12, 3.0],
                 np.float32)
    assert T.tf32_rna(x).tolist() == [1.0 + 2.0 ** -10, 1.0 + 2.0 ** -9, -(1.0 + 2.0 ** -10), 1.0, 3.0]


def test_cases_cover_every_axis():
    simt_d = {c.d for c in T.CASES}
    tc_d = {c.d for c in T.CASES if T.tc_ok(c.d)}
    assert set(T.SIMT_D) <= simt_d and set(T.TC_D) <= tc_d
    for kern in ('simt', 'tc'):
        rows = {c.n_rows for c in T.CASES if kern in c.kernels}
        Ns = {c.N for c in T.CASES if kern in c.kernels}
        assert set(T.ROWS) <= rows, kern
        assert set(T.NS) <= Ns, kern
        assert any(c.N == c.n_items for c in T.CASES if kern in c.kernels)
        assert any(c.n_items < T.TC_HALF for c in T.CASES if kern in c.kernels)
        assert {round(c.rated_value, 1) == 2.5 for c in T.CASES if kern in c.kernels} == {True, False}
    for c in T.CASES:                                        # ids stay inside the tables: a bad id is a device fault
        assert c.users.min() >= 0 and c.users.max() < c.U.shape[0]
        assert c.cols.size == 0 or (c.cols.min() >= 0 and c.cols.max() < c.n_items)
        assert len(c.rowptr) == c.U.shape[0] + 1
        for u in range(c.U.shape[0]):
            assert np.all(np.diff(c.cols[c.rowptr[u]:c.rowptr[u + 1]]) > 0)     # sorted, distinct
    # rated values above, below and between the scores, and 0
    assert any(c.rated_value > np.abs(T.scores64(c.U, c.V, np.unique(c.users))).max() for c in T.CASES)
    assert any(c.rated_value < -np.abs(T.scores64(c.U, c.V, np.unique(c.users))).max() for c in T.CASES)


def test_cases_reach_every_branch_of_both_kernels():
    """Computed from the kernel constants: each branch where the selection can go wrong is taken by some case."""
    simt, tc = set(), set()
    for c in T.CASES:
        simt |= T.simt_paths(c)
        if T.tc_ok(c.d):
            tc |= T.tc_paths(c)
    assert {'compact', 'compact_tie_at_cut', 'cta_tail', 'tile_tail', 'k_tail', 'k_full', 'k_chunks', 'rated_rescued',
            'rated_demoted'} <= simt, simt
    assert {'kb1', 'kb2', 'k_pad', 'compact', 'tie_search', 'compact_final', 'tie_search_final', 'cta_tail',
            'quarter_tail', 'empty_quarter', 'half_tail', 'group_tail', 'empty_half', 'second_list_empty', 'open_row',
            'rated_rescued', 'sig_saturated', 'sig_false_hit'} <= tc, tc


@pytest.mark.parametrize('family', sorted(T.FAMILY_TARGETS))
def test_every_defect_is_told_apart_by_its_families(family):
    cases = [c for c in T.CASES if c.family == family]
    assert cases
    for defect in T.FAMILY_TARGETS[family]:
        assert defect in T.DEFECTS
        assert any(not T.same_output(*T.defect_output(c, defect)) for c in cases), (family, defect)


def test_heap_survivors_at_a_tie():
    """find_k_largest at a tie across the cut: of the tied items the heap keeps the largest ids among those up to the
    N-th item (in id order) scoring at least the cut -- not the smallest ids, which the kernel contract keeps."""
    from qrec_b200.util.qmath import find_k_largest
    s = np.full(8, -4.0)
    s[[5, 6]] = 0.0
    ids, vals = find_k_largest(3, s)
    assert sorted(ids[:2]) == [5, 6] and ids[2] == 2 and vals == [0.0, 0.0, -4.0]    # kernel contract: 5, 6, 0
    s = np.full(400, -4.0)
    s[100:110] = -2.0
    ids, _ = find_k_largest(12, s)
    assert sorted(ids[:10]) == list(range(100, 110)) and sorted(ids[10:]) == [10, 11]  # kernel contract: 0, 1
    # when a tie straddles the cut, the same as the kernel contract: the earliest ids scoring at least the cut
    s = np.full(12, -4.0)
    s[6:] = -2.0
    ids, _ = find_k_largest(3, s)
    assert sorted(ids) == [6, 7, 8]


# ---------------------------------------------------------------------------------------------------------------------
# the `-eval gpu` driver on numpy stand-ins of the kernels it calls
def _engine_stand_ins(monkeypatch, calls):
    import torch
    from qrec_b200 import engine as E

    def score_topn(U, V, user_ids, rated_rowptr, rated_cols, N, rated_value=0.0, out_ids=None, out_scores=None,
                   tensor_cores=None):
        assert 1 <= N <= min(T.NMAX, V.shape[0])
        calls.append(N)
        ids, s = T.topn(U.numpy(), V.numpy(), user_ids.numpy(), rated_rowptr.numpy(), rated_cols.numpy(), N,
                        rated_value)
        return torch.from_numpy(ids.astype(np.int32)), torch.from_numpy(s)

    def sgemm(A, B, C, trans_a=False, trans_b=False, alpha=1.0, beta=0.0):
        assert trans_b and not trans_a and alpha == 1.0 and beta == 0.0
        C.copy_(torch.from_numpy((A.numpy().astype(np.float64) @ B.numpy().astype(np.float64).T).astype(np.float32)))
        return C

    def mask_rated(scores, users, rowptr, cols, value=0.0):
        m = T.rated_mask(rowptr.numpy(), cols.numpy(), users.numpy(), scores.shape[1])
        scores[torch.from_numpy(m)] = value
        return scores

    monkeypatch.setattr(E, 'score_topn', score_topn)
    monkeypatch.setattr(E, 'sgemm', sgemm)
    monkeypatch.setattr(E, 'mask_rated', mask_rated)


def _csr(case):
    from types import SimpleNamespace
    return SimpleNamespace(sorted_rowptr=case.rowptr, sorted_cols=case.cols)


@pytest.mark.parametrize('case', T.CASES, ids=repr)
def test_batched_top_n_returns_the_reference_heap_lists(case, monkeypatch):
    import torch
    from qrec_b200.evaluate import batched_top_n
    calls = []
    _engine_stand_ins(monkeypatch, calls)
    N = T.driver_n(case)
    block = max(1, case.n_rows // 3)                         # several blocks per user list
    ids, vals = batched_top_n(torch.from_numpy(case.U), torch.from_numpy(case.V), case.users, _csr(case), N,
                              block=block)
    ref_i, ref_s = T.heap_reference(case)
    assert ids.shape == ref_i.shape and ids.dtype == np.int64 and vals.dtype == np.float32
    bad = [r for r in range(case.n_rows) if not np.array_equal(ids[r], ref_i[r])]
    assert not bad, 'rows %s: %s != heap %s' % (bad[:5], ids[bad[0]].tolist(), ref_i[bad[0]].tolist())
    assert np.array_equal(vals, ref_s)
    assert len(calls) == -(-case.n_rows // block)


def test_batched_top_n_takes_n_up_to_100(monkeypatch):
    import torch
    from qrec_b200.evaluate import batched_top_n
    _engine_stand_ins(monkeypatch, [])
    case = next(c for c in T.CASES if c.N == 101 and c.n_items > 101)
    for N in (0, 101):
        with pytest.raises(ValueError):
            batched_top_n(torch.from_numpy(case.U), torch.from_numpy(case.V), case.users, _csr(case), N)


@pytest.mark.parametrize('d', [3, 8])
def test_eval_gpu_writes_the_host_flow_lines(d, monkeypatch, tmp_path):
    """evalRanking with `engine=-eval gpu` (the driver over the kernel contract) and without it write the same
    recommendation lines and measure lines, on scores whose ties the kernel contract orders differently."""
    monkeypatch.chdir(tmp_path)
    host = T.tie_model(d, str(tmp_path), 'cpu', gpu_eval=False)
    _engine_stand_ins(monkeypatch, [])
    dev = T.tie_model(d, str(tmp_path), 'cpu', gpu_eval=True)
    assert dev.recOutput == host.recOutput and dev.measure == host.measure
    csr = host.data.rated_csr()
    users = np.array([host.data.user[u] for u in host.data.testSet_u], np.int32)
    args = (host.P, host.Q, users, csr.sorted_rowptr, csr.sorted_cols, 10)
    assert not T.same_output(T.topn(*args, 0.0), T.heap_topn(*args))
