#!/usr/bin/env python
"""K2 decomposed on the bipartite blocks of the benchmark graph (1M users x 100K items x 50M edges, d=64): the user-side
product A_ui E_i (gathers from the 25.6 MB item block), the item-side product A_iu E_u (gathers from the 256 MB user
block) and the item side cut into column blocks of users so that one block of E_u fits the L2
(parallel.split_csr_columns / blocked_spmm), each with the row-split product spmm_csr(..., rowsplit=True).  One JSON
line per measurement.

  python tools/bench_spmm_blocks.py [--blocks 2 3 4 6 8] [--steps 10]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--blocks', type=int, nargs='+', default=[2, 3, 4, 6, 8])
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    import torch
    from qrec_b200 import engine as E, synthetic, parallel
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    U, I, DEG, D = 1_000_000, 100_000, 50, 64
    data = synthetic.make_interactions(U, I, DEG, device=dev)
    rp, co, va = synthetic.build_norm_adj(data, U, I, dev)
    A_ui, A_iu, _ = parallel.shard_bipartite_by_user(rp, co, va, U, I, 0, 1)
    del rp, co, va
    g = torch.Generator(device=dev); g.manual_seed(0)
    Eu = torch.randn(U, D, device=dev, generator=g) * 0.005
    Ei = torch.randn(I, D, device=dev, generator=g) * 0.005
    Yu, Yi, Si = torch.empty_like(Eu), torch.empty_like(Ei), torch.empty_like(Ei)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    def spmm(A, X, Y, acc=None, s=0.0):
        return E.spmm_csr(A[0], A[1], A[2], X, Y, acc=acc, acc_scale=s, rowsplit=True)

    nnz = int(A_ui[1].numel())
    ms_u = timed(lambda: spmm(A_ui, Ei, Yu))
    print(json.dumps({'product': 'user side A_ui E_i', 'rows': U, 'nnz': nnz, 'ms': ms_u,
                      'G_gathers_per_s': nnz / ms_u / 1e6}), flush=True)
    ms_i = timed(lambda: spmm(A_iu, Eu, Yi))
    print(json.dumps({'product': 'item side A_iu E_u', 'blocks': 1, 'rows': I, 'nnz': nnz, 'ms': ms_i,
                      'G_gathers_per_s': nnz / ms_i / 1e6}), flush=True)
    ref = Yi.clone()
    for nb in args.blocks:
        blocks = parallel.split_csr_columns(A_iu, U, nb)
        ms = timed(lambda: parallel.blocked_spmm(spmm, blocks, Eu, Yi, Si, None, 0.0))
        err = float((Yi - ref).abs().max() / ref.abs().max())
        print(json.dumps({'product': 'item side A_iu E_u', 'blocks': nb, 'block_MB': U / nb * D * 4 / 1e6,
                          'ms': ms, 'G_gathers_per_s': nnz / ms / 1e6, 'rel_err_vs_unblocked': err}), flush=True)
        del blocks
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
