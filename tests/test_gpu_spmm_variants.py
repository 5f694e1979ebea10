"""Experimental row-split SpMM configurations (csrc/spmm_variants.cu) against the production kernel:
they change the number of outstanding gathers and the occupancy, not the floating-point order, so the
outputs must be bit-identical.  Needs a GPU."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('variant', range(7))
def test_variant_reproduces_production_bits(variant):
    import scipy.sparse as sp
    import torch
    from qrec_b200 import engine as E
    rng = np.random.default_rng(variant)
    n, m, d = 3000, 2500, 64
    A = sp.random(n, m, density=0.01, format='lil', dtype=np.float32, random_state=variant)
    A[5, :] = 0                                               # empty row
    A[7, :600] = rng.random(600).astype(np.float32)           # long row: many index chunks
    for k, ln in enumerate((1, 3, 4, 5, 8, 9, 15, 16, 17, 31, 32, 33)):      # every group / chunk boundary
        A[20 + k, :] = 0
        A[20 + k, :ln] = rng.random(ln).astype(np.float32) + 0.1
    A = A.tocsr(); A.sort_indices()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
    rp, co, va = dev(A.indptr.astype(np.int64)), dev(A.indices.astype(np.int32)), dev(A.data.astype(np.float32))
    X = torch.randn(m, d, device='cuda')
    Y0, Y1 = torch.full((n, d), float('nan'), device='cuda'), torch.full((n, d), float('nan'), device='cuda')
    acc0 = torch.randn(n, d, device='cuda'); acc1 = acc0.clone()
    E.spmm_csr(rp, co, va, X, Y0, acc=acc0, acc_scale=0.25, rowsplit=True)
    E.spmm_csr_rowsplit_variant(variant, rp, co, va, X, Y1, acc=acc1, acc_scale=0.25)
    torch.cuda.synchronize()
    assert torch.equal(Y0, Y1) and torch.equal(acc0, acc1)
    assert float(Y1[5].abs().sum()) == 0.0
    E.spmm_csr_rowsplit_variant(variant, rp, co, va, X, Y1)                # without the fused accumulation
    assert torch.equal(Y0, Y1)


def test_variant_entry_point_limits():
    import torch
    from qrec_b200 import engine as E
    rp = torch.zeros(3, dtype=torch.int64, device='cuda'); co = torch.zeros(0, dtype=torch.int32, device='cuda')
    va = torch.zeros(0, device='cuda')
    with pytest.raises(E.QRecError):
        E.spmm_csr_rowsplit_variant(7, rp, co, va, torch.zeros(4, 64, device='cuda'), torch.zeros(2, 64, device='cuda'))
    with pytest.raises(E.QRecError):
        E.spmm_csr_rowsplit_variant(0, rp, co, va, torch.zeros(4, 32, device='cuda'), torch.zeros(2, 32, device='cuda'))
