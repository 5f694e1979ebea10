"""K5 v2 (persistent, TMA-fed, warp-specialised wgmma GEMM) against an fp64 product and against v1.
A is consumed as raw fp32 bits (TF32 truncation: up to 2^-10 per operand, one-sided), so the bound is
twice v1's.  Needs a GPU."""
import os

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


def _bound(A, B_kn):
    return (A.double().abs() @ B_kn.double().abs()) * 2.0 ** -8 + 1e-6


def test_exact_on_tf32_representable_inputs(torch, E):
    """Small integers are exact in TF32: the product must be bit exact, which pins the tensor map, the
    swizzle, the descriptors, the stage ring and the epilogue transpose (any
    misplaced element is a wrong integer).  Sizes cover several row tiles per CTA and ragged edges."""
    g = torch.Generator(device='cuda'); g.manual_seed(0)
    for M, N, K in ((384, 192, 160), (128, 64, 32), (100000, 320, 128), (129, 65, 68), (1, 1, 4), (4097, 130, 320)):
        A = torch.randint(-8, 9, (M, K), device='cuda', generator=g).float()
        W = torch.randint(-8, 9, (K, N), device='cuda', generator=g).float()
        C = torch.full((M, N), float('nan'), device='cuda')
        E.tc_gemm_v2(A, W, C)
        assert torch.equal(C.double(), A.double() @ W.double()), (M, N, K)
        C.fill_(float('nan'))
        E.tc_gemm_v2(A, W.t().contiguous(), C, b_is_nk=True)
        assert torch.equal(C.double(), A.double() @ W.double()), (M, N, K)


@pytest.mark.parametrize('M,N,K', [(128, 64, 32), (256, 128, 128), (10240, 320, 128), (200, 100, 36), (327680, 320, 128),
                                   (10240, 160, 320), (10240, 64, 128)])
def test_forward_layout_bias_relu(torch, E, M, N, K):
    g = torch.Generator(device='cuda'); g.manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, device='cuda', generator=g)
    W = torch.randn(K, N, device='cuda', generator=g) * 0.2
    b = torch.randn(N, device='cuda', generator=g)
    C = torch.full((M, N), float('nan'), device='cuda')
    E.tc_gemm_v2(A, W, C)
    assert bool(((C.double() - A.double() @ W.double()).abs() <= _bound(A, W)).all())
    E.tc_gemm_v2(A, W, C, epilogue=E.EPI_BIAS_RELU, bias=b)
    ref = torch.relu(A.double() @ W.double() + b.double())
    assert bool(((C.double() - ref).abs() <= _bound(A, W)).all())
    C1 = torch.empty_like(C)
    E.tc_gemm(A, W, C1, epilogue=E.EPI_BIAS_RELU, bias=b)                # v1: same product, rna-rounded A
    assert bool(((C - C1).abs().double() <= _bound(A, W)).all())


@pytest.mark.parametrize('M,N,K', [(128, 64, 32), (10240, 128, 320), (10240, 320, 128), (77, 130, 64)])
def test_backward_data_layout_relu_mask(torch, E, M, N, K):
    g = torch.Generator(device='cuda'); g.manual_seed(M + N + K)
    dY = torch.randn(M, K, device='cuda', generator=g)
    W = torch.randn(N, K, device='cuda', generator=g) * 0.2
    H = torch.randn(M, N, device='cuda', generator=g)
    C = torch.empty(M, N, device='cuda')
    E.tc_gemm_v2(dY, W, C, b_is_nk=True, epilogue=E.EPI_RELU_MASK, mask=H)
    ref = (dY.double() @ W.double().t()) * (H > 0).double()
    assert bool(((C.double() - ref).abs() <= _bound(dY, W.t())).all())


def test_limits(torch, E):
    with pytest.raises(E.QRecError):                                      # K beyond the resident B block
        E.tc_gemm_v2(torch.zeros(8, 324, device='cuda'), torch.zeros(324, 8, device='cuda'), torch.zeros(8, 8, device='cuda'))
    C = torch.zeros(0, 8, device='cuda')
    E.tc_gemm_v2(torch.zeros(0, 8, device='cuda'), torch.zeros(8, 8, device='cuda'), C)   # M = 0: no launch
