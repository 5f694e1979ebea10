#!/usr/bin/env python
"""LightGCN-path microbench at the synthetic scale (1M users x 100K items x 50M edges, d=64):
K2 SpMM alone, and full LightGCN minibatch steps (reference semantics: whole propagation, its
backward and a dense Adam for every minibatch).  Prints one JSON line per measurement.

  python tools/bench_graph.py [--layers 3] [--batch 2048 65536] [--steps 10] [--scale 1.0]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, default=3)
    ap.add_argument('--batch', type=int, nargs='+', default=[2048, 65536])
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--scale', type=float, default=1.0)
    ap.add_argument('--zipf', action='store_true')
    ap.add_argument('--spmm-only', action='store_true')
    args = ap.parse_args()
    import torch
    from qrec_b200 import engine as E, synthetic
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    U, I, DEG, D = int(1_000_000 * args.scale), int(100_000 * args.scale), 50, 64
    data = synthetic.make_interactions(U, I, DEG, device=dev, zipf=args.zipf)
    rowptr, cols, vals = synthetic.build_norm_adj(data, U, I, dev)
    N, nnz = U + I, int(cols.numel())
    peak = 6540.5
    try:
        peak = float(json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'])
    except Exception:
        pass
    g = torch.Generator(device=dev); g.manual_seed(0)
    X = torch.randn(N, D, device=dev, generator=g) * 0.005
    Y = torch.empty_like(X)
    acc = torch.zeros_like(X)

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps

    algo = nnz * (8 + 4 * D) + N * (4 + 4 * D)            # SURVEY 8(d): no-reuse gather model
    floor = nnz * 8 + N * (4 + 8 * D)
    for rowsplit in (False, True):
        ms = timed(lambda: E.spmm_csr(rowptr, cols, vals, X, Y, acc=acc, acc_scale=0.25, rowsplit=rowsplit), args.steps, args.warmup)
        print(json.dumps({'kernel': 'spmm_csr_rowsplit_f32(+acc)' if rowsplit else 'spmm_csr_f32(+acc, nnz-balanced)',
                          'rows': N, 'nnz': nnz, 'd': D, 'ms': ms, 'algorithmic_GB': algo / 1e9,
                          'achieved_GBs': algo / ms / 1e6, 'frac_of_measured_hbm': algo / ms / 1e6 / peak,
                          'compulsory_GB': floor / 1e9, 'zipf': args.zipf}))
    if args.spmm_only:
        return
    # full LightGCN steps through the drop-in class's step function
    from qrec_b200.base.graphRecommender import DeviceCSR
    from qrec_b200.model.ranking.LightGCN import LightGCN

    class Shell(LightGCN):            # engine state only; no Rating object needed for the step
        def __init__(self):
            pass
    m = Shell()
    m.num_users, m.num_items, m.emb_size, m.emb_pad, m.n_layers = U, I, D, D, args.layers
    m.lRate, m.regU, m.device = 0.001, 0.001, dev
    m.norm_adj = DeviceCSR.from_tensors((N, N), rowptr, cols, vals)
    m.norm_adj.rowsplit = not args.zipf
    m.ego = X.clone()
    m.user_embeddings, m.item_embeddings = m.ego[:U], m.ego[U:]
    m._buf = [torch.empty(N, D, device=dev) for _ in range(2)]
    m._mean, m._grad, m._total = torch.empty(N, D, device=dev), torch.zeros(N, D, device=dev), torch.empty(N, D, device=dev)
    m._adam_m, m._adam_v = torch.zeros(N, D, device=dev), torch.zeros(N, D, device=dev)
    m._loss, m._step = torch.zeros(1, dtype=torch.float64, device=dev), 0
    perm = torch.randperm(U * DEG, device=dev, generator=g)
    for B in args.batch:
        idx = perm[:B]
        bu, bi = data['u'][idx].contiguous(), data['i'][idx].contiguous()
        bj = E.sample_neg_philox(bu, data['sorted_rowptr'], data['sorted_cols'], I, 1, 0)
        ms = timed(lambda: m.train_step(bu, bi, bj), args.steps, args.warmup)
        steps_per_epoch = -(-U * DEG // B)
        step_bytes = 2 * args.layers * algo + (args.layers + 2) * N * D * 4 * 2 + B * (3 * 4 * D * 2 + 12) + 7 * N * D * 4
        print(json.dumps({'lightgcn_step_ms': ms, 'batch': B, 'layers': args.layers, 'steps_per_epoch': steps_per_epoch,
                          'epoch_s_extrapolated': ms * steps_per_epoch / 1e3, 'loss': float(m._loss.item()),
                          'algorithmic_GB_per_step': step_bytes / 1e9, 'frac_of_measured_hbm': step_bytes / ms / 1e6 / peak}))


if __name__ == '__main__':
    main()
