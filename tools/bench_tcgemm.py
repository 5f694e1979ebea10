#!/usr/bin/env python
"""Times the wgmma TF32 GEMM on NeuMF's MLP shapes (d=64): forward [B,128]x[128,320],
[B,320]x[320,128], [B,128]x[128,64] and the backward-data products, B = 5*batch_size samples."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from qrec_b200 import engine as E
    peak = 1656.8
    try:
        peak = float(json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['bf16_tflops'])
    except Exception:
        pass
    g = torch.Generator(device='cuda'); g.manual_seed(0)
    for B in (10240, 327680):
        for (K, N, nk) in ((128, 320, False), (320, 128, False), (128, 64, False), (64, 128, True), (128, 320, True), (320, 128, True)):
            A = torch.randn(B, K, device='cuda', generator=g)
            W = torch.randn((N, K) if nk else (K, N), device='cuda', generator=g)
            bias = torch.randn(N, device='cuda', generator=g)
            C = torch.empty(B, N, device='cuda')
            fn = ((lambda: E.tc_gemm(A, W, C, b_is_nk=True)) if nk
                  else (lambda: E.tc_gemm(A, W, C, epilogue=E.EPI_BIAS_RELU, bias=bias)))
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(20):
                fn()
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / 20
            flops = 2.0 * B * K * N
            bytes_ = 4.0 * (B * K + K * N + B * N)
            print(json.dumps({'kernel': 'tc_gemm_tf32', 'M': B, 'N': N, 'K': K, 'b_is_nk': nk, 'ms': ms,
                              'TFLOPs': flops / ms / 1e9, 'GBs': bytes_ / ms / 1e6,
                              'note': 'tf32 dense peak is half the bf16 peak (%.0f TF/s measured bf16)' % peak}))


if __name__ == '__main__':
    main()
