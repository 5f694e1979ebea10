"""The kernels that opt in to more than 48 KB of dynamic shared memory, run on two GPUs in one process: the opt-in
is a property of the kernel as loaded on each device, so it has to be made again on the second device.  Device 0
first, then device 1: the NeuMF GEMM (tc_gemm, bias + ReLU epilogue, 50 KB) and the tensor-core top-N, each
against a torch / numpy reference at the tolerances of test_gpu_tcgemm.py and test_gpu_topn.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two visible GPUs')
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def _topn_reference(P, Q, users, rp, co, N):
    ids, vals = [], []
    for u in users:
        s = (Q.astype(np.float64) @ P[u].astype(np.float64)).astype(np.float32)
        s[co[rp[u]:rp[u + 1]]] = 0.0
        top = np.lexsort((np.arange(len(s)), -s))[:N]
        ids.append(top); vals.append(s[top])
    return np.array(ids), np.array(vals)


def test_dynamic_smem_kernels_on_two_devices_in_one_process(torch, E):
    rng = np.random.default_rng(3)
    nu, ni, d, N = 200, 1500, 64, 20
    P = rng.standard_normal((nu, d)).astype(np.float32)
    Q = rng.standard_normal((ni, d)).astype(np.float32)
    deg = rng.integers(0, 40, nu)
    rp = np.zeros(nu + 1, np.int64); rp[1:] = np.cumsum(deg)
    co = np.concatenate([np.sort(rng.choice(ni, k, replace=False)) for k in deg]).astype(np.int32)
    users = rng.permutation(nu)[:150].astype(np.int32)
    rid, rval = _topn_reference(P, Q, users, rp, co, N)
    for dev in (0, 1):
        with torch.cuda.device(dev):
            g = torch.Generator(device='cuda'); g.manual_seed(11)
            A = torch.randn(300, 96, device='cuda', generator=g)
            W = torch.randn(96, 130, device='cuda', generator=g) * 0.2
            b = torch.randn(130, device='cuda', generator=g)
            C = torch.full((300, 130), float('nan'), device='cuda')
            E.tc_gemm(A, W, C, epilogue=E.EPI_BIAS_RELU, bias=b)
            ref = torch.relu(A.double() @ W.double() + b.double())
            bound = (A.double().abs() @ W.double().abs()) * 2.0 ** -9 + 1e-6
            assert bool(((C.double() - ref).abs() <= bound).all()), 'tc_gemm on cuda:%d' % dev

            cuda = lambda a: torch.from_numpy(a).cuda()   # noqa: E731
            ids, vals = E.score_topn(cuda(P), cuda(Q), cuda(users), cuda(rp), cuda(co), N, tensor_cores=True)
            torch.cuda.synchronize()
            ids, vals = ids.cpu().numpy(), vals.cpu().numpy()
            np.testing.assert_allclose(vals, rval, rtol=2e-5, atol=2e-5, err_msg='score_topn on cuda:%d' % dev)
            for r in range(len(users)):
                gap_ok = np.ones(N, bool)
                gap_ok[1:] &= (rval[r, :-1] - rval[r, 1:]) > 1e-4
                gap_ok[:-1] &= (rval[r, :-1] - rval[r, 1:]) > 1e-4
                assert np.array_equal(ids[r][gap_ok], rid[r][gap_ok]), 'score_topn on cuda:%d, row %d' % (dev, r)
