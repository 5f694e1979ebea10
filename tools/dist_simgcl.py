#!/usr/bin/env python
"""BASELINE config 5 under torchrun (one rank per GPU, NCCL): SimGCL (LightGCN encoders + InfoNCE, d=64) with
the user table row-sharded over the ranks and the item table replicated (parallel.UserShardedSimGCL).
 (1) parity: the sharded step equals the single-GPU drop-in SimGCL step on a down-scaled graph (same Philox
     noise, same losses, same gradients, same tables after Adam);
 (2) timing: `--users-per-gpu` x world users, `--items` items, degree 50 -- with 8 GPUs and the defaults this is
     the 10M users x 1M items x 500M interactions of BASELINE.json configs[4].

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/dist_simgcl.py
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
    ap.add_argument('--layers', type=int, default=2)            # config/SimGCL.conf:11 -n_layer 2
    ap.add_argument('--batch', type=int, default=2048)
    ap.add_argument('--users-per-gpu', type=int, default=1_250_000)
    ap.add_argument('--items', type=int, default=1_000_000)
    ap.add_argument('--skip-parity', action='store_true')
    ap.add_argument('--skip-timing', action='store_true')
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    import bench
    from qrec_b200 import engine as E, synthetic, parallel
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (('RANK', 0), ('WORLD_SIZE', 1), ('LOCAL_RANK', 0)))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev, pg_options=dist.ProcessGroupNCCL.Options(is_high_priority_stream=True))
    D, DEG = 64, 50
    CL, EPS = 0.5, 0.1                                             # config/SimGCL.conf:11 -lambda 0.5 -eps 0.1
    g = torch.Generator(device=dev); g.manual_seed(11)

    # ---------------- parity on a small graph (every rank also runs the 1-GPU step)
    if not args.skip_parity:
        U, I = 16000, 1600
        data = synthetic.make_interactions(U, I, DEG, device=dev)           # same seed on every rank
        rp, co, va = synthetic.build_norm_adj(data, U, I, dev)
        g3 = torch.Generator(device=dev); g3.manual_seed(3)
        ego = (torch.rand(U + I, D, device=dev, generator=g3) * 2 - 1) * 0.02
        A_ui, A_iu, (lo, hi) = parallel.shard_bipartite_by_user(rp, co, va, U, I, rank, world)
        m = parallel.UserShardedSimGCL(A_ui, A_iu, ego[lo:hi].clone(), ego[U:].clone(), args.layers, 0.001, 0.001, lo, U, CL, EPS,
                                       noise_seed=0x5151, d_valid=D)
        from qrec_b200.base.graphRecommender import DeviceCSR
        from qrec_b200.model.ranking.SimGCL import SimGCL

        class Shell(SimGCL):
            def __init__(self):
                pass
        ref = Shell()
        ref.num_users, ref.num_items, ref.emb_size, ref.emb_pad, ref.n_layers = U, I, D, D, args.layers
        ref.lRate, ref.regU, ref.device, ref.cl_rate, ref.eps = 0.001, 0.001, dev, CL, EPS
        N = U + I
        ref.norm_adj, ref.ego = DeviceCSR.from_tensors((N, N), rp, co, va), ego.clone()
        ref._buf = [torch.empty(N, D, device=dev) for _ in range(2)]
        ref._main = torch.empty(N, D, device=dev)
        ref._pert = [torch.empty(N, D, device=dev) for _ in range(2)]
        ref._grad, ref._total = torch.zeros(N, D, device=dev), torch.zeros(N, D, device=dev)
        ref._adam_m, ref._adam_v = torch.zeros(N, D, device=dev), torch.zeros(N, D, device=dev)
        ref._loss, ref._step, ref.noise_seed = torch.zeros(2, dtype=torch.float64, device=dev), 0, 0x5151
        mine = torch.cat([torch.arange(lo, hi, device=dev), torch.arange(U, U + I, device=dev)])
        for step in range(3):
            idx = torch.randint(0, U * DEG, (args.batch,), device=dev, generator=g)
            bu, bi = data['u'][idx].contiguous(), data['i'][idx].contiguous()
            bj = E.sample_neg_philox(bu, data['sorted_rowptr'], data['sorted_cols'], I, 1, step)
            ref.train_step(bu, bi, bj)
            m.train_step(bu, bi, bj)
            _, rec_ref, cl_ref = ref.losses()
            _, rec, cl = m.losses()
            assert abs(rec - rec_ref) <= 1e-5 * abs(rec_ref) and abs(cl - cl_ref) <= 1e-5 * abs(cl_ref), (rec, rec_ref, cl, cl_ref)
            gtot = torch.cat([m.tot_u, m.tot_i])
            gref = ref._total[mine]
            assert float((gtot - gref).abs().max()) <= 2e-3 * float(gref.abs().max()), 'gradient mismatch'
            torch.testing.assert_close(torch.cat([m.Eu, m.Ei]), ref.ego[mine], rtol=2e-3, atol=2e-4)
        if world > 1:                                         # the replicated item rows stay bit-identical across ranks
            chk = [torch.empty_like(m.Ei) for _ in range(world)]
            dist.all_gather(chk, m.Ei)
            assert all(torch.equal(chk[0], c) for c in chk), 'replicated item rows diverged'
        if rank == 0:
            print(json.dumps({'parity': 'UserShardedSimGCL == single-GPU SimGCL step (3 steps: losses 1e-5, gradients 2e-3 of max, '
                                        'tables; item replicas bit-identical)', 'world': world, 'graph': [U, I, U * DEG]}))
        del data, rp, co, va, ego, m, ref, A_ui, A_iu
        torch.cuda.empty_cache()

    # ---------------- timing at config 5's per-GPU scale
    if not args.skip_timing:
        UL, I = args.users_per_gpu, args.items
        U = UL * world
        data = synthetic.make_interactions(UL, I, DEG, device=dev, user_offset=rank * UL, seed=515)
        bench.NUM_USERS, bench.NUM_ITEMS = U, I
        A_ui, A_iu = bench.local_bipartite_blocks(torch, dist, data, UL, I, world)
        gi = torch.Generator(device=dev); gi.manual_seed(7)
        bound_i = (6.0 / (I + D)) ** 0.5                           # xavier on [rows, d] (SimGCL.py:42-44)
        Ei = (torch.rand(I, D, device=dev, generator=gi) * 2 - 1) * bound_i      # same seed: replicated
        gi.manual_seed(70 + rank)
        Eu = (torch.rand(UL, D, device=dev, generator=gi) * 2 - 1) * (6.0 / (U + D)) ** 0.5
        m = parallel.UserShardedSimGCL(A_ui, A_iu, Eu, Ei, args.layers, 0.001, 0.001, rank * UL, U, CL, EPS, d_valid=D)
        per_rank = args.batch // world
        batches = []
        for t in range(args.steps + 2):
            idx = torch.randint(0, UL * DEG, (per_rank,), device=dev, generator=g)
            bu_l, bi = data['u'][idx].contiguous(), data['i'][idx].contiguous()
            bj = E.sample_neg_philox(bu_l, data['sorted_rowptr'], data['sorted_cols'], I, 1, t)
            b = torch.stack([(bu_l + rank * UL).int(), bi, bj])
            if world > 1:
                parts = [torch.empty_like(b) for _ in range(world)]
                dist.all_gather(parts, b)
                b = torch.cat(parts, dim=1)
            batches.append(tuple(b[k].contiguous() for k in range(3)))
        for t in range(2):
            m.train_step(*batches[t])
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for t in range(args.steps):
            m.train_step(*batches[2 + t])
        b.record()
        torch.cuda.synchronize()
        tt = torch.tensor([a.elapsed_time(b) / args.steps], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        total, rec, cl = m.losses()
        if rank == 0:
            ms = float(tt.item())
            nnz = 2 * U * DEG
            layer_passes = 4 * args.layers                       # 3 encoders + 1 collapsed backward
            print(json.dumps({
                'config': 'SimGCL (LightGCN encoders + InfoNCE), d=64, n_layers=%d, %d users x %d items x %d interactions, '
                          'user table row-sharded over %d GPU(s), item table replicated' % (args.layers, U, I, U * DEG, world),
                'world': world, 'batch': args.batch, 'step_ms': ms, 'steps_per_epoch': -(-U * DEG // args.batch),
                'epoch_s_at_batch': ms * (-(-U * DEG // args.batch)) / 1e3,
                'layer_passes_per_step': layer_passes, 'spmm_nnz_per_pass_whole_job': nnz,
                'item_block_allreduce_MB_per_pass': I * D * 4 / 1e6,
                'spmm_algorithmic_GBs_whole_job': layer_passes * (nnz * (8 + 4 * D) + (U + I) * (4 + 4 * D)) / (ms * 1e-3) / 1e9,
                'losses': {'total': total, 'rec': rec, 'cl': cl}}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
