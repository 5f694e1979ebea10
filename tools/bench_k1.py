#!/usr/bin/env python
"""K1 variants on the benchmark workload (50 M triples, 1M x 100K, d=64): the user-major epoch with given and with
fused-sampled negatives, the stand-alone sampler, and the batch kernel on shuffled triples.  One JSON line each."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from qrec_b200 import engine as E, synthetic
    dev = torch.device('cuda', 0)
    U, I, DEG, D = 1_000_000, 100_000, 50, 64
    data = synthetic.make_interactions(U, I, DEG, device=dev)
    P, Q = synthetic.init_tables(U, I, D, device=dev)
    g = torch.Generator(device=dev); g.manual_seed(1)
    perm = torch.randperm(U * DEG, device=dev, generator=g)
    u, i = data['u'][perm].contiguous(), data['i'][perm].contiguous()
    j = E.sample_neg_philox(u, data['sorted_rowptr'], data['sorted_cols'], I, 1, 0)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    # user-major (reference order): CSR positives, negatives sampled in the same order
    ju = E.sample_neg_philox(data['u'], data['sorted_rowptr'], data['sorted_cols'], I, 1, 0)
    rowptr = data['sorted_rowptr']
    for name, fn in (('usermajor(P in registers)', lambda: E.bpr_sgd_usermajor(P, Q, rowptr, data['i'], ju, 0.01, 0.001, 0.001, loss)),
                     ('batch kernel on user-major order', lambda: E.bpr_sgd_batch(P, Q, data['u'], data['i'], ju, 0.01, 0.001, 0.001, loss))):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 10
        print(json.dumps({'k1_variant': name, 'ms_per_50M': ms, 'G_triples_s': 50 / ms, 'algorithmic_TBs': 50e6 * 1548 / ms / 1e9}))
    # fused sampling, without / with the signature pre-test (the latter only once validated on hardware)
    seeds = iter(range(1000))
    fused = [('fused sampling', lambda: E.bpr_epoch_usermajor(P, Q, rowptr, data['i'], data['sorted_rowptr'], data['sorted_cols'],
                                                            I, 1, next(seeds), 0.01, 0.001, 0.001, loss))]
    if True:
        sig = E.rated_signature(data['sorted_rowptr'], data['sorted_cols'])
        fused.append(('fused sampling + signature pre-test',
                      lambda: E.bpr_epoch_usermajor_sig(P, Q, rowptr, data['i'], data['sorted_rowptr'], data['sorted_cols'], sig,
                                                        I, 1, next(seeds), 0.01, 0.001, 0.001, loss)))
    for name, fn in fused:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 10
        print(json.dumps({'k1_variant': name, 'ms_per_50M': ms, 'G_triples_s': 50 / ms}))
    for fn_name, fn in (('sampler shuffled order', lambda: E.sample_neg_philox(u, data['sorted_rowptr'], data['sorted_cols'], I, 1, 0, out=j)),
                        ('sampler user-major order', lambda: E.sample_neg_philox(data['u'], data['sorted_rowptr'], data['sorted_cols'], I, 1, 0, out=ju))):
        fn(); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            fn()
        b.record()
        torch.cuda.synchronize()
        print(json.dumps({'kernel': fn_name, 'ms_per_50M': a.elapsed_time(b) / 10}))
    for _ in range(3):
        E.bpr_sgd_batch(P, Q, u, i, j, 0.01, 0.001, 0.001, loss)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        E.bpr_sgd_batch(P, Q, u, i, j, 0.01, 0.001, 0.001, loss)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 10
    print(json.dumps({'k1_variant': 'red', 'ms_per_50M': ms, 'G_triples_s': 50 / ms, 'algorithmic_TBs': 50e6 * 1548 / ms / 1e9}))


if __name__ == '__main__':
    main()
