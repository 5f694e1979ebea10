"""Both K8 kernels (csrc/topn_kernels.cu, csrc/topn_tc.cu) and the `-eval gpu` ranking (evaluate.batched_top_n) on every
exact-score case of topn_cases.py: ids and scores bit for bit, no gap mask.  The kernels keep the kernel contract
(score descending, id ascending, one zero); batched_top_n returns util.qmath.find_k_largest's lists."""
import numpy as np
import pytest

import topn_cases as T

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


KERNEL_CASES = [pytest.param(c, k, id='%s-%s' % (k, c.name)) for c in T.CASES for k in c.kernels]


@pytest.mark.parametrize('case,kernel', KERNEL_CASES)
def test_kernel_equals_kernel_reference(torch, E, case, kernel):
    n, N = case.n_rows, case.N
    out_ids = torch.full((n, N), T.SENTINEL_ID, dtype=torch.int32, device='cuda')
    out_scores = _dev(torch, np.full((n, N), T.SENTINEL_BITS, np.uint32).view(np.float32))
    E.score_topn(_dev(torch, case.U), _dev(torch, case.V), _dev(torch, case.users), _dev(torch, case.rowptr),
                 _dev(torch, case.cols), N, rated_value=case.rated_value, out_ids=out_ids, out_scores=out_scores,
                 tensor_cores=(kernel == 'tc'))
    torch.cuda.synchronize()
    ids, bits = out_ids.cpu().numpy(), out_scores.cpu().numpy().view(np.uint32)
    assert not np.any(ids == T.SENTINEL_ID) and not np.any(bits == T.SENTINEL_BITS), 'unwritten output'
    ref_i, ref_s = T.kernel_reference(case)
    bad = [r for r in range(n) if not np.array_equal(ids[r], ref_i[r])]
    assert not bad, 'rows %s: %s != %s' % (bad[:5], ids[bad[0]].tolist(), ref_i[bad[0]].tolist())
    assert np.array_equal(bits, ref_s.view(np.uint32))


@pytest.mark.parametrize('case', T.CASES, ids=repr)
def test_batched_top_n_equals_heap_reference(torch, case):
    from types import SimpleNamespace
    from qrec_b200.evaluate import batched_top_n
    csr = SimpleNamespace(sorted_rowptr=case.rowptr, sorted_cols=case.cols)
    ids, vals = batched_top_n(_dev(torch, case.U), _dev(torch, case.V), case.users, csr, T.driver_n(case),
                              block=max(1, case.n_rows // 3))
    ref_i, ref_s = T.heap_reference(case)
    bad = [r for r in range(case.n_rows) if not np.array_equal(ids[r], ref_i[r])]
    assert not bad, 'rows %s: %s != heap %s' % (bad[:5], ids[bad[0]].tolist(), ref_i[bad[0]].tolist())
    assert np.array_equal(vals, ref_s)             # by value: the heap compares -0.0 and +0.0 equal


@pytest.mark.parametrize('d', [3, 8])
def test_eval_gpu_writes_the_host_flow_lines(torch, d, monkeypatch, tmp_path):
    """evalRanking with and without `engine=-eval gpu` (d = 8: the tensor-core kernel, d = 3: the SIMT kernel) writes
    the same recommendation and measure lines, with ties inside the top-10 lists and across their cut."""
    monkeypatch.chdir(tmp_path)
    host = T.tie_model(d, str(tmp_path), 'cuda', gpu_eval=False)
    dev = T.tie_model(d, str(tmp_path), 'cuda', gpu_eval=True)
    assert dev.recOutput == host.recOutput and dev.measure == host.measure
    csr = host.data.rated_csr()
    users = np.array([host.data.user[u] for u in host.data.testSet_u], np.int32)
    args = (host.P, host.Q, users, csr.sorted_rowptr, csr.sorted_cols, 10)
    assert not T.same_output(T.topn(*args, 0.0), T.heap_topn(*args))     # the kernel contract alone would differ
