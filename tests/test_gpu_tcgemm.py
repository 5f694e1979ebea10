"""K5 building block: the wgmma TF32 GEMM against an fp64 product.  TF32 keeps 10 mantissa
bits of each operand, so the tolerance is 2^-10-ish relative to |A||B| row/column norms."""
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


def _check(torch, C, ref, A, B_kn):
    bound = (A.double().abs() @ B_kn.double().abs()) * 2.0 ** -9 + 1e-6
    assert bool(((C.double() - ref).abs() <= bound).all()), float(((C.double() - ref).abs() / bound).max())


@pytest.mark.parametrize('M,N,K', [(128, 64, 32), (128, 64, 64), (256, 128, 128), (10240, 320, 128), (200, 100, 36),
                                   (1, 1, 4), (129, 65, 68), (10240, 64, 128), (327680, 320, 128), (10240, 160, 320)])
def test_forward_layout_bias_relu(torch, E, M, N, K):
    g = torch.Generator(device='cuda'); g.manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, device='cuda', generator=g)
    W = torch.randn(K, N, device='cuda', generator=g) * 0.2
    b = torch.randn(N, device='cuda', generator=g)
    C = torch.full((M, N), float('nan'), device='cuda')
    E.tc_gemm(A, W, C)
    _check(torch, C, A.double() @ W.double(), A, W)
    E.tc_gemm(A, W, C, epilogue=E.EPI_BIAS_RELU, bias=b)
    ref = torch.relu(A.double() @ W.double() + b.double())
    bound = (A.double().abs() @ W.double().abs()) * 2.0 ** -9 + 1e-6
    assert bool(((C.double() - ref).abs() <= bound).all())


@pytest.mark.parametrize('M,N,K', [(128, 64, 32), (10240, 128, 320), (10240, 320, 128), (77, 130, 64)])
def test_backward_data_layout_relu_mask(torch, E, M, N, K):
    """dX = (dY @ W^T) * (H > 0) with W stored [N_out_of_this_gemm, K] = [K_in, N_out]."""
    g = torch.Generator(device='cuda'); g.manual_seed(M + N + K)
    dY = torch.randn(M, K, device='cuda', generator=g)
    W = torch.randn(N, K, device='cuda', generator=g) * 0.2           # [N,K] row-major
    H = torch.randn(M, N, device='cuda', generator=g)
    C = torch.empty(M, N, device='cuda')
    E.tc_gemm(dY, W, C, b_is_nk=True)
    _check(torch, C, dY.double() @ W.double().t(), dY, W.t())
    E.tc_gemm(dY, W, C, b_is_nk=True, epilogue=E.EPI_RELU_MASK, mask=H)
    ref = (dY.double() @ W.double().t()) * (H > 0).double()
    bound = (dY.double().abs() @ W.double().abs().t()) * 2.0 ** -9 + 1e-6
    assert bool(((C.double() - ref).abs() <= bound).all())


def test_exact_on_tf32_representable_inputs(torch, E):
    """Small integers are exact in TF32 and fp32 accumulation: the product must be bit exact,
    which pins the descriptor/swizzle plumbing (any misplaced element shows up as a wrong integer)."""
    g = torch.Generator(device='cuda'); g.manual_seed(0)
    A = torch.randint(-8, 9, (384, 160), device='cuda', generator=g).float()
    W = torch.randint(-8, 9, (160, 192), device='cuda', generator=g).float()
    C = torch.empty(384, 192, device='cuda')
    E.tc_gemm(A, W, C)
    assert torch.equal(C, A @ W) or torch.equal(C.double(), A.double() @ W.double())
    Wt = W.t().contiguous()
    E.tc_gemm(A, Wt, C, b_is_nk=True)
    assert torch.equal(C.double(), A.double() @ W.double())
