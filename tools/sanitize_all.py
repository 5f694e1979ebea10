#!/usr/bin/env python
"""Launches every kernel of libqrec.so once at small sizes -- meant to run under
  compute-sanitizer --tool memcheck|racecheck|synccheck python tools/sanitize_all.py
(SURVEY.md section 5: the reference has no sanitizer story; K1 throughput mode is racy by design
through atomics only, everything else must be clean)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from qrec_b200 import engine as E, parallel
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
    nu, ni, d, n = 300, 400, 64, 1000
    u = rng.integers(0, nu, n).astype(np.int32); i = rng.integers(0, ni, n).astype(np.int32)
    j = ((i + 1 + rng.integers(0, ni - 1, n)) % ni).astype(np.int32)
    P, Q = dev((rng.random((nu, d)) / 3).astype(np.float32)), dev((rng.random((ni, d)) / 3).astype(np.float32))
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    csr = E.RatedCSR(nu, ni, u, i)
    jj = E.sample_neg_philox(dev(u), dev(csr.sorted_rowptr), dev(csr.sorted_cols), ni, 1, 0)
    E.bpr_sgd_batch(P, Q, dev(u), dev(i), jj, 0.01, 0.001, 0.001, loss)
    for dd in (8, 48, 128, 256):
        Pd, Qd = torch.rand(nu, dd, device='cuda'), torch.rand(ni, dd, device='cuda')
        E.bpr_sgd_batch(Pd, Qd, dev(u), dev(i), dev(j), 0.01, 0.001, 0.001, loss)
    wu, wi, wj = E.bpr_order_prepare(u, i, j, nu, ni)
    for dt in (torch.float32, torch.float64):
        E.bpr_sgd_ordered(P.to(dt), Q.to(dt), dev(u), dev(i), dev(j), dev(wu), dev(wi), dev(wj), 0.01, 0.001, 0.001, loss)
    E.sumsq(P, loss); E.sumsq(P.double(), loss)
    pipe = E.HostPipeline(0, chunk_triples=300)
    pipe.bpr_epoch(P, Q, u, i, j, 0.01, 0.001, 0.001); pipe.close()
    m = parallel.ShardedItemTableBPR(P, Q, ni, 0, 1, 0.01, 0.001, 0.001)
    m.step(dev(u), dev(i), dev(j))
    # graph path
    import scipy.sparse as sp
    N = nu + ni
    A = sp.random(N, N, density=0.02, format='csr', dtype=np.float32, random_state=1); A.sort_indices()
    rp, co, va = dev(A.indptr.astype(np.int64)), dev(A.indices.astype(np.int32)), dev(A.data)
    X, Y, acc = torch.rand(N, d, device='cuda'), torch.empty(N, d, device='cuda'), torch.zeros(N, d, device='cuda')
    for rs in (False, True):
        E.spmm_csr(rp, co, va, X, Y, acc=acc, acc_scale=0.5, rowsplit=rs)
    gU, gV = torch.zeros_like(P), torch.zeros_like(Q)
    E.bpr_grad_scatter(P, Q, dev(u), dev(i), dev(j), 1e-7, 0.001, gU, gV, loss)
    E.adam_dense_tf1(P, torch.zeros_like(P), torch.zeros_like(P), gU, 0.001, 1)
    E.axpby(Y, X, acc, 1.0, 2.0)
    # K6 / dense
    E.simgcl_perturb(X, 0.1, 7, 1, 1, acc=acc, acc_scale=0.5, d_valid=62)
    idx = dev(rng.permutation(N)[:129].astype(np.int32))
    Z, nrm = torch.empty(129, d, device='cuda'), torch.empty(129, device='cuda')
    E.gather_normalize(X, idx, Z, nrm)
    S = torch.empty(129, 129, device='cuda')
    E.sgemm(Z, Z, S, trans_b=True)
    E.infonce_rows(S, 0.2, loss)
    dZ = torch.empty_like(Z)
    E.sgemm(S, Z, dZ); E.sgemm(S, Z, dZ, trans_a=True)
    E.normalize_bwd_scatter(dZ, Z, nrm, idx, 0.5, acc)
    W = torch.rand(d, d, device='cuda')
    big = torch.rand(5000, d, device='cuda')
    E.sgemm(big, big, W, trans_a=True)                    # split-K path
    H, out, norms = torch.empty(N, d, device='cuda'), torch.empty(N, 3 * d, device='cuda'), torch.empty(N, device='cuda')
    E.ngcf_act_fwd(X, 0.9, 1, 3, 0, 1, H, out[:, d:2 * d], norms)
    E.ngcf_act_bwd(out[:, d:2 * d], None, H, X, norms, 0.9, 1, 3, 0, 1, Y)
    E.mul(Y, X, acc)
    # K5
    B = 300
    A0 = torch.rand(B, 128, device='cuda'); W1 = torch.rand(128, 320, device='cuda'); b1 = torch.rand(320, device='cuda')
    H1 = torch.empty(B, 320, device='cuda')
    E.tc_gemm(A0, W1, H1, epilogue=E.EPI_BIAS_RELU, bias=b1)
    dX = torch.empty(B, 128, device='cuda')
    E.tc_gemm(H1, W1, dX, b_is_nk=True, epilogue=E.EPI_RELU_MASK, mask=A0)
    uu, ii = dev(u[:B]), dev(i[:B])
    X0 = torch.empty(B, 2 * d, device='cuda')
    E.gather_rows(P, uu, X0[:, :d]); E.gather_rows(Q, ii, X0[:, d:])
    E.scatter_add_rows(gU, uu, X0[:, :d])
    y, dz = torch.empty(B, device='cuda'), torch.empty(B, device='cuda')
    UG, IG, H3 = (torch.rand(B, d, device='cuda') for _ in range(3))
    GMF, dUG, dIG, dH3 = (torch.empty(B, d, device='cuda') for _ in range(4))
    hm, hl = torch.rand(d, device='cuda'), torch.rand(d, device='cuda')
    r = (torch.rand(B, device='cuda') > 0.8).float()
    for mode in (0, 1, 2):
        E.neumf_head(mode, 1, UG, IG, H3, hm, hl, r, 0.001, loss, y, dz, GMF, dUG, dIG, dH3)
    sc = torch.rand(64, ni, device='cuda')
    E.mask_rated(sc, dev(np.arange(64, dtype=np.int32)), dev(csr.sorted_rowptr), dev(csr.sorted_cols))
    torch.cuda.synchronize()
    print('sanitize_all: launched', E.launch_count(), 'kernels')
    if True:
        # K9 (rating-prediction MF): kept apart until its first hardware run has passed
        n9 = n
        u9, i9 = np.ascontiguousarray(u[:n9]), np.ascontiguousarray(i[:n9])
        r9 = torch.rand(n9, device='cuda') * 4
        wu9, wi9 = E.mf_order_prepare(u9, i9, nu, ni)
        Bu, Bi = torch.zeros(nu, device='cuda'), torch.zeros(ni, device='cuda')
        for kind in (0, 1, 2):
            E.mf_sgd_batch(kind, P, Q, dev(u9), dev(i9), r9, 0.01, 0.01, 0.01, loss, Bu, Bi, 0.01, 2.0)
            E.mf_sgd_ordered(kind, P, Q, dev(u9), dev(i9), r9, dev(wu9), dev(wi9), 0.01, 0.01, 0.01, loss, Bu, Bi, 0.01, 2.0)
        E.mf_sgd_ordered(E.EE_RATINGS, P, Q, dev(u9), dev(i9), r9, dev(wu9), dev(wi9), 0.01, 0.01, 0.01, loss, Bu, Bi,
                         0.01, 2.0)
        E.mf_predict_pairs(P, Q, dev(u9), dev(i9), Bu, Bi, 2.0)
        sig = E.rated_signature(dev(csr.sorted_rowptr), dev(csr.sorted_cols))
        E.bpr_epoch_usermajor_sig(P, Q, dev(csr.pos_rowptr), dev(csr.pos_cols), dev(csr.sorted_rowptr),
                                  dev(csr.sorted_cols), sig, ni, 5, 0, 0.01, 0.001, 0.001, loss)
        torch.cuda.synchronize()
        print('sanitize_all: + K9, launched', E.launch_count(), 'kernels')
        # round-2 kernels
        from qrec_b200.graph_build import JointAdjacency
        E.bpr_epoch_usermajor(P, Q, dev(csr.pos_rowptr), dev(csr.pos_cols), dev(csr.sorted_rowptr), dev(csr.sorted_cols), ni, 5, 0,
                              0.01, 0.001, 0.001, loss)
        ids, vals = E.score_topn(P, Q, dev(np.arange(nu, dtype=np.int32)), dev(csr.sorted_rowptr), dev(csr.sorted_cols), 10)
        J = JointAdjacency(dev(u.astype(np.int64)), dev(i.astype(np.int64)), nu, ni, device='cuda')
        J.full(); J.edge_dropout(0.3, 1, 2, 3)
        Bt, Dt, St = Q.clone(), torch.empty(Q.numel(), device='cuda'), torch.empty(Q.numel(), device='cuda')
        E.table_delta(Q.view(-1), Bt.view(-1), Dt, St)
        E.table_reduce_scatter_p2p([Dt.data_ptr(), Dt.data_ptr()], 1, St, Dt.numel())
        E.table_gather_merge_p2p([St.data_ptr(), St.data_ptr()], Q.view(-1), Bt.view(-1), Dt)
        E.table_merge(Q.view(-1), Bt.view(-1), Dt, St)
        E.ubench_row_ops(torch.rand(1000, 64, device='cuda'), 5000, 2)
        cnt, snd = torch.empty(2, dtype=torch.int32, device='cuda'), torch.empty(2 * 900, dtype=torch.int32, device='cuda')
        pos, ovf = torch.empty(n, dtype=torch.int32, device='cuda'), torch.zeros(1, dtype=torch.int32, device='cuda')
        E.bucket_requests(dev(i), ni // 2, 2, 900, cnt, snd, pos, ovf)
        E.simgcl_perturb(X, 0.1, 7, 1, 1, acc=acc, acc_scale=0.5, d_valid=62, row_offset=12345)
        torch.cuda.synchronize()
        print('sanitize_all: + round 2, launched', E.launch_count(), 'kernels')
        # K10 (WRMF): Gram + row solve, both table types, the one-tile-per-thread and three-tiles-per-thread builds, with
        # whole and padded tiles (d = 37: NT = 1, four groups; d = 97: NT = 3, two groups)
        rp_u = torch.from_numpy(np.bincount(u, minlength=nu).cumsum()).cuda()
        rowptr = torch.cat([torch.zeros(1, dtype=torch.int64, device='cuda'), rp_u])
        cols = dev(i[np.argsort(u, kind='stable')])
        order = dev(E.als_row_order(rowptr.cpu().numpy()))
        for dd in (20, 37, 97, 128):
            for dt in (torch.float64, torch.float32):
                Xs, Ys = torch.rand(nu, dd, device='cuda', dtype=dt), torch.rand(ni, dd, device='cuda', dtype=dt)
                G = E.als_gram(Ys)
                E.als_solve_rows(Xs, Ys, G, rowptr, cols, torch.ones(n, device='cuda', dtype=dt), 1.0, 10.0, order,
                                 loss=loss)
        torch.cuda.synchronize()
        print('sanitize_all: + K10, launched', E.launch_count(), 'kernels')
        # K11 (SVD++): the ordered kernel (both table types, one staged chunk and several) and the user-major epoch
        # at every lane-group width, one user in flight and a full grid
        rv = torch.rand(n, device='cuda') * 4
        for dd, dt in ((10, torch.float64), (256, torch.float64), (37, torch.float32)):
            T = [torch.rand(nu, dd, device='cuda', dtype=dt), torch.rand(ni, dd, device='cuda', dtype=dt),
                 torch.rand(ni, dd, device='cuda', dtype=dt), torch.rand(nu, device='cuda', dtype=dt),
                 torch.rand(ni, device='cuda', dtype=dt)]
            E.svdpp_sgd_ordered(*T, dev(np.sort(u)), cols, rv.to(dt), rowptr, cols, 0.01, 0.01, 0.01, 0.1, 0.01, 3.0,
                                loss)
        for dd in (4, 32, 64, 128):
            T = [torch.rand(nu, dd, device='cuda'), torch.rand(ni, dd, device='cuda'), torch.rand(ni, dd, device='cuda'),
                 torch.rand(nu, device='cuda'), torch.rand(ni, device='cuda')]
            for k in (1, 0):
                E.svdpp_epoch_usermajor(*T, rowptr, cols, rv, order, 0.01, 0.01, 0.01, 0.1, 0.01, 3.0, loss,
                                        max_users_in_flight=k)
        torch.cuda.synchronize()
        print('sanitize_all: + K11, launched', E.launch_count(), 'kernels')
        # K12 (CoFactor): both co-occurrence passes (and so the SPPMI), then the item sweep for both table types and
        # both tile builds, over the SPPMI of the same interactions
        pairs = np.unique(np.stack([i, u]), axis=1)                              # distinct (item, user), item-major
        irp = torch.from_numpy(np.concatenate([[0], np.bincount(pairs[0], minlength=ni).cumsum()])).cuda()
        icol = dev(pairs[1].astype(np.int32))
        srp, scol, sval = E.sppmi_csr(irp, icol, nu, 5, 0)
        for dd in (20, 37, 97, 128):
            for dt in (torch.float64, torch.float32):
                Y, G = torch.rand(ni, dd, device='cuda', dtype=dt), torch.rand(ni, dd, device='cuda', dtype=dt)
                w, c = torch.rand(ni, device='cuda', dtype=dt), torch.rand(ni, device='cuda', dtype=dt)
                Xs = torch.rand(nu, dd, device='cuda', dtype=dt)
                E.cofactor_item_sweep(Y, G, w, c, Xs, E.als_gram(Xs), (irp, icol, torch.ones_like(icol, dtype=dt)),
                                      (srp, scol, sval.to(dt)), 1.0, 1.0, 10.0)
        torch.cuda.synchronize()
        print('sanitize_all: + K12, launched', E.launch_count(), 'kernels', 'SPPMI nnz', scol.shape[0])
        # K13 (ExpoMF): the user half (mu by column) and the item half with the prior (mu by row), for both tile
        # builds, over the same interactions (users with no entries included)
        for dd in (20, 37, 97, 128):
            th, be = torch.rand(nu, dd, device='cuda') * 0.1, torch.rand(ni, dd, device='cuda') * 0.1
            mu, mu_out = torch.full((ni,), 0.01, device='cuda'), torch.empty(ni, device='cuda')
            E.expomf_half_epoch(th, be, rowptr, cols, mu, False, 1e-5, 1.0, order)
            E.expomf_half_epoch(be, th, irp, icol, mu, True, 1e-5, 1.0, dev(E.als_row_order(irp.cpu().numpy())),
                                mu_out=mu_out)
        torch.cuda.synchronize()
        print('sanitize_all: + K13, launched', E.launch_count(), 'kernels')
        # K14 (SERec): both halves with the uniform first-epoch prior and with the social prior from A and deg (users
        # of degree 0 included), the item half with the fused sums, for both tile builds; then the square case, whose
        # item half reads the prior with its rows as users, over the entries of the first nu items
        deg = torch.randint(0, 40, (nu,), dtype=torch.int32, device='cuda') * (torch.rand(nu, device='cuda') < 0.5)
        iord = dev(E.als_row_order(irp.cpu().numpy()))
        for dd in (20, 37, 97, 128):
            th, be = torch.rand(nu, dd, device='cuda') * 0.1, torch.rand(ni, dd, device='cuda') * 0.1
            A, A_out = None, torch.empty(ni, dtype=torch.float64, device='cuda')
            for _ in range(2):
                E.serec_half_epoch(th, be, rowptr, cols, A, deg, True, 1e-3, 0.01, order)
                E.serec_half_epoch(be, th, irp, icol, A, deg, False, 1e-3, 0.01, iord, asum_out=A_out)
                A, A_out = A_out, torch.empty_like(A_out)
        rp_h, col_h = rowptr.cpu().numpy(), cols.cpu().numpy()
        keep = col_h < nu
        sq_rp = np.concatenate([[0], np.cumsum(np.bincount(np.repeat(np.arange(nu), np.diff(rp_h))[keep], minlength=nu))])
        sq_rp, sq_col = dev(sq_rp.astype(np.int64)), dev(col_h[keep].astype(np.int32))
        sq = torch.rand(nu, 20, device='cuda') * 0.1
        A_sq = torch.rand(nu, dtype=torch.float64, device='cuda') * 10
        E.serec_half_epoch(sq, torch.rand(nu, 20, device='cuda') * 0.1, sq_rp, sq_col, A_sq, deg, True, 1e-3, 0.01,
                           dev(E.als_row_order(sq_rp.cpu().numpy())), asum_out=torch.empty_like(A_sq))
        torch.cuda.synchronize()
        print('sanitize_all: + K14, launched', E.launch_count(), 'kernels')
        # K15 (UserKNN / ItemKNN / SlopeOne): neighbour lists of every metric over the user rows (cold queries
        # included), K past the candidate lists, the predictions, and SlopeOne's fused launch on one CTA and on many
        up = np.unique(np.stack([u, i]), axis=1)                                 # distinct (user, item), user-major
        rp_h = np.concatenate([[0], np.bincount(up[0], minlength=nu).cumsum()]).astype(np.int64)
        krp, kcol = dev(rp_h), dev(up[1].astype(np.int32))
        kv = dev((np.arange(up.shape[1]) % 9 + 1).astype(np.float64) / 2)
        km = dev(np.bincount(up[0], weights=kv.cpu().numpy(), minlength=nu) / np.maximum(np.diff(rp_h), 1))
        kq = dev(np.concatenate([np.arange(0, nu, 7), [-1, -1]]).astype(np.int32))
        for metric in (0, 1, 2):
            ksq = dev(E.knn_squares(rp_h, kv.cpu().numpy(), km.cpu().numpy(), metric))
            for K in (20, nu + 5):
                out = E.knn_neighbours(krp, kcol, kv, ksq, km, ni, kq, metric, K)
            lq = dev(np.arange(kq.shape[0], dtype=np.int32))
            E.knn_predict(krp, *E.knn_sorted_view(krp, kcol, kv), km, 3.0, kq, *out, lq, dev(np.full(kq.shape[0], 1, np.int32)), True)
        ikv = torch.full((icol.shape[0],), 3.5, dtype=torch.float64, device='cuda')
        ikm = torch.full((ni,), 3.5, dtype=torch.float64, device='cuda')
        titems = dev(np.concatenate([np.arange(0, ni, 5), [-1]]).astype(np.int32))
        for c in (1, 0):
            E.slopeone_predict(irp, icol, ikv, ikm, krp, kcol, kv, km, 3.0, titems,
                               dev((np.arange(300) % titems.shape[0]).astype(np.int32)),
                               dev((np.arange(300) % nu).astype(np.int32)), max_ctas=c)
        torch.cuda.synchronize()
        print('sanitize_all: + K15, launched', E.launch_count(), 'kernels')
        # K17 (SocialMF / SoReg / SREE user pass) on a ring-with-chords trust graph with self-follows, every kind and
        # both dtypes, one CTA and a full grid; SoReg's pair similarities over the K15 user rows
        fol = [sorted({(a + 1) % nu, (7 * a + 3) % nu, a}) for a in range(nu)]
        frp = np.concatenate([[0], np.cumsum([len(x) for x in fol])]).astype(np.int64)
        fcol = np.array([v for x in fol for v in x], np.int32)
        back = np.argsort(fcol, kind='stable')
        grp = np.concatenate([[0], np.cumsum(np.bincount(fcol, minlength=nu))]).astype(np.int64)
        gcol = np.repeat(np.arange(nu, dtype=np.int32), np.diff(frp))[back]
        visit = np.random.default_rng(4).permutation(nu)[: nu - 3].astype(np.int32)
        spos, _ = E.social_order_prepare(visit, nu, frp, fcol, grp, gcol)
        for dt in (torch.float64, torch.float32):
            vals = torch.rand(fcol.shape[0], device='cuda').to(dt)
            for kind in (0, 1):
                for nw in (1, 0):
                    E.social_user_pass(kind, torch.rand(nu, 33, device='cuda').to(dt), dev(visit), dev(spos), dev(frp),
                                       dev(fcol), vals, dev(grp), dev(gcol), vals[torch.from_numpy(back).cuda()], 0.05,
                                       0.1, torch.zeros(1, dtype=torch.float64, device='cuda'), n_warps=nw)
                E.sree_user_pass(torch.rand(nu, 33, device='cuda').to(dt), dev(visit), dev(spos), dev(frp), dev(fcol),
                                 vals, dev(grp), dev(gcol), 0.05, 0.5, torch.zeros(1, dtype=torch.float64, device='cuda'),
                                 n_warps=nw)
        ksq = dev(E.knn_squares(rp_h, kv.cpu().numpy(), km.cpu().numpy(), 0))
        pa = dev(np.arange(0, nu, 3).astype(np.int32))
        E.knn_pair_similarity(krp, kcol, kv, ksq, km, *E.knn_sorted_view(krp, kcol, kv),
                              E.knn_sorted_view(krp, kcol, ksq)[1], pa, (pa * 5 + 1) % nu,
                              torch.ones(pa.shape[0], dtype=torch.float64, device='cuda'))
        torch.cuda.synchronize()
        print('sanitize_all: + K17 and the pair similarities, launched', E.launch_count(), 'kernels')


if __name__ == '__main__':
    main()
