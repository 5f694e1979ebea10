#!/usr/bin/env python
"""Sharded LightGCN step under torchrun (one rank per GPU, NCCL): (1) parity against the single-GPU
step on a down-scaled graph, (2) step time on the synthetic 1M x 100K x 50M-edge graph.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/dist_lightgcn.py
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--layers', type=int, default=3)
    ap.add_argument('--batch', type=int, default=2048)
    ap.add_argument('--item-blocks', type=int, default=1, help='column blocks of the item-side SpMM (experimental)')
    ap.add_argument('--scheme', default='user', choices=['user', 'rows', 'cols'],
                    help='user: users partitioned + items replicated (all-reduce of the item block per layer); '
                         'rows: all rows partitioned (all-gather of the whole table per layer); '
                         'cols: embedding columns partitioned, adjacency replicated (one [B] all-reduce per step)')
    ap.add_argument('--skip-parity', action='store_true', help='timing part only')
    ap.add_argument('--profile-range', action='store_true', help='cudaProfilerStart/Stop around the timed steps (ncu --profile-from-start off)')
    ap.add_argument('--graph', action='store_true', help='scheme user: replay the step from a CUDA graph (train_step_graphed)')
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    from qrec_b200 import engine as E, synthetic, parallel
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (('RANK', 0), ('WORLD_SIZE', 1), ('LOCAL_RANK', 0)))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    D, DEG = 64, 50

    def build(U, I):
        data = synthetic.make_interactions(U, I, DEG, device=dev)           # same seed on every rank
        rp, co, va = synthetic.build_norm_adj(data, U, I, dev)
        g = torch.Generator(device=dev); g.manual_seed(3)
        ego = torch.randn(U + I, D, device=dev, generator=g) * 0.005
        if args.scheme == 'cols':
            from qrec_b200.base.graphRecommender import DeviceCSR
            dw = D // world
            part, mine = None, None
            m = parallel.ColumnShardedLightGCN(DeviceCSR.from_tensors((U + I, U + I), rp, co, va),
                                               ego[:, rank * dw:(rank + 1) * dw].contiguous(), U, args.layers, 0.001, 0.001)
            m.local_nnz = int(co.numel())
        elif args.scheme == 'rows':
            part = parallel.NodePartition(U, I, world)
            lrp, lco, lva = parallel.shard_adjacency(rp, co, va, part, rank)
            mine = part.local_nodes(rank).to(dev)
            m = parallel.ShardedLightGCN(part, rank, lrp, lco, lva, ego[mine].contiguous(), args.layers, 0.001, 0.001)
        else:
            A_ui, A_iu, (lo, hi) = parallel.shard_bipartite_by_user(rp, co, va, U, I, rank, world)
            part = None
            mine = torch.cat([torch.arange(lo, hi, device=dev), torch.arange(U, U + I, device=dev)])
            m = parallel.UserShardedLightGCN(A_ui, A_iu, ego[lo:hi].clone(), ego[U:].clone(), args.layers, 0.001, 0.001, lo,
                                             item_side_blocks=args.item_blocks)
            m.local_nnz = int(A_ui[1].numel()) * 2
        return data, (rp, co, va), ego, part, mine, m

    if not args.skip_parity:
        parity(args, build, rank, world, dev, D, DEG, E, torch)
    timing(args, build, rank, world, dev, D, DEG, E, torch, dist)
    if world > 1:
        if parallel.any_rank_captured_graphs():
            parallel.finish_process(0)      # a live CUDA graph with NCCL work inside blocks the communicator teardown
        dist.destroy_process_group()


def parity(args, build, rank, world, dev, D, DEG, E, torch):
    # ---------------- parity on a small graph (every rank also runs the 1-GPU step)
    U, I = 16000, 1600
    data, (rp, co, va), ego, part, mine, m = build(U, I)
    from qrec_b200.base.graphRecommender import DeviceCSR
    from qrec_b200.model.ranking.LightGCN import LightGCN

    class Shell(LightGCN):
        def __init__(self):
            pass
    ref = Shell()
    ref.num_users, ref.num_items, ref.emb_size, ref.emb_pad, ref.n_layers, ref.lRate, ref.regU, ref.device = U, I, D, D, args.layers, 0.001, 0.001, dev
    N = U + I
    ref.norm_adj, ref.ego = DeviceCSR.from_tensors((N, N), rp, co, va), ego.clone()
    ref._buf = [torch.empty(N, D, device=dev) for _ in range(2)]
    ref._mean, ref._grad, ref._total = (torch.zeros(N, D, device=dev) for _ in range(3))
    ref._adam_m, ref._adam_v = torch.zeros(N, D, device=dev), torch.zeros(N, D, device=dev)
    ref._loss, ref._step = torch.zeros(1, dtype=torch.float64, device=dev), 0
    g = torch.Generator(device=dev); g.manual_seed(11)
    for step in range(3):
        idx = torch.randint(0, U * DEG, (args.batch,), device=dev, generator=g)
        bu, bi = data['u'][idx].contiguous(), data['i'][idx].contiguous()
        bj = E.sample_neg_philox(bu, data['sorted_rowptr'], data['sorted_cols'], I, 1, step)
        l_ref = ref.train_step(bu, bi, bj).item()
        l = (m.train_step_graphed if args.graph else m.train_step)(bu, bi, bj).item()     # graph: eager, capture + replay, replay
        assert abs(l - l_ref) <= 1e-5 * abs(l_ref), (l, l_ref)
        if args.scheme == 'cols':
            lo_c = rank * (D // world)
            got, gtot = m.ego, m.total
            gref, eref = ref._total[:, lo_c:lo_c + D // world], ref.ego[:, lo_c:lo_c + D // world]
        else:
            got = m.ego if args.scheme == 'rows' else torch.cat([m.Eu, m.Ei])
            gtot = m.total if args.scheme == 'rows' else torch.cat([m.tot_u, m.tot_i])
            gref, eref = ref._total[mine], ref.ego[mine]
        # gradients first (Adam's first steps turn a tiny gradient difference into a visible table
        # difference wherever |g| ~ eps, so the tables get a looser absolute tolerance)
        assert float((gtot - gref).abs().max()) <= 2e-3 * float(gref.abs().max()), 'gradient mismatch'
        torch.testing.assert_close(got, eref, rtol=2e-3, atol=2e-4)
    if args.graph:
        assert m.graph_error is None and any(st['graph'] is not None for st in m._graphs.values()), m.graph_error
    if rank == 0:
        print(json.dumps({'parity': 'sharded (%s%s) == single-GPU LightGCN step' % (args.scheme, ', CUDA graph' if args.graph else ''),
                          'world': world, 'graph': [U, I, U * DEG]}))
    del data, rp, co, va, ego, m, ref
    torch.cuda.empty_cache()


def timing(args, build, rank, world, dev, D, DEG, E, torch, dist):
    # ---------------- timing at the benchmark scale
    U, I = 1_000_000, 100_000
    g = torch.Generator(device=dev)
    data, (rp, co, va), ego, part, mine, m = build(U, I)
    del rp, co, va, ego
    torch.cuda.empty_cache()
    g.manual_seed(12)                                  # every rank draws the same minibatch (the cols scheme requires it)
    idx = torch.randint(0, U * DEG, (args.batch,), device=dev, generator=g)
    bu, bi = data['u'][idx].contiguous(), data['i'][idx].contiguous()
    bj = E.sample_neg_philox(bu, data['sorted_rowptr'], data['sorted_cols'], I, 1, 0)
    step_fn = m.train_step_graphed if args.graph else m.train_step
    for _ in range(2):
        step_fn(bu, bi, bj)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if args.profile_range:
        torch.cuda.profiler.start()
    a.record()
    for _ in range(args.steps):
        step_fn(bu, bi, bj)
    b.record()
    torch.cuda.synchronize()
    if args.profile_range:
        torch.cuda.profiler.stop()
    t = torch.tensor([a.elapsed_time(b) / args.steps], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        ms = float(t.item())
        print(json.dumps({'lightgcn_sharded_step_ms': ms, 'world': world, 'layers': args.layers, 'batch': args.batch,
                          'epoch_s_at_batch': ms * (-(-U * DEG // args.batch)) / 1e3, 'scheme': args.scheme,
                          'cuda_graph': bool(args.graph and getattr(m, 'graph_error', None) is None),
                          'graph_error': getattr(m, 'graph_error', None),
                          'local_nnz': int(m.cols.numel()) if args.scheme == 'rows' else m.local_nnz}))


if __name__ == '__main__':
    main()
