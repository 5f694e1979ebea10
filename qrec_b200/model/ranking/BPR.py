"""BPR-MF on the H100 engine -- drop-in for model/ranking/BPR.py of the reference.

`trainModel` replaces the numpy loop (BPR.py:19-43): every epoch the (u,i,j) stream is produced
by the bit-exact C clone of Python's MT19937 sampler (continuing from the interpreter's global
`random` state, so `random.seed(s)` gives the reference's triples), then
  * engine -mode parity : qrec_bpr_sgd_ordered_{f64,f32} -- sequential-equivalent SGD, the same
                          P/Q as the reference after every epoch;
  * engine -mode fast   : qrec_bpr_sgd_usermajor_f32 -- the fused throughput kernel in the same
                          user-major order (P[u] sequential inside a user, item rows scatter-added).
`trainModel_tf` replaces the TF1 Adam graph (BPR.py:77-96) with K3 + full-table L2 + K4.
"""
import random

import numpy as np

from ...base.iterativeRecommender import IterativeRecommender


class BPR(IterativeRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(BPR, self).__init__(conf, trainingSet, testSet, fold)

    def initModel(self):
        super(BPR, self).initModel()

    def trainModel(self):
        import torch
        from ... import engine as E
        print('Preparing item sets...')
        csr = self.data.rated_csr()
        dev = self._device()
        fast = self.engine_mode == 'fast'
        d = self.emb_size
        P, Q = self._upload(self.P, dev, pad=True), self._upload(self.Q, dev, pad=True)
        acc = torch.zeros(3, dtype=torch.float64, device=dev)
        mt = E.MT19937()
        print('training...')
        epoch = 0
        while epoch < self.maxEpoch:
            mt.setstate(random.getstate())
            u, i, j = mt.sample_bpr_epoch(csr)               # BPR.py:31-38
            random.setstate(mt.getstate())
            du, di, dj = (torch.from_numpy(x).to(dev) for x in (u, i, j))
            acc.zero_()
            if fast and P.shape[1] <= 128:
                # the sampler's stream is user-major (BPR.py:31-33): P[u] stays in registers per user
                E.bpr_sgd_usermajor(P, Q, torch.from_numpy(csr.pos_rowptr).to(dev), di, dj, self.lRate, self.regU,
                                    self.regI, acc[0:1])
            elif fast:
                E.bpr_sgd_batch(P, Q, du, di, dj, self.lRate, self.regU, self.regI, acc[0:1])
            else:
                wu, wi, wj = E.bpr_order_prepare(u, i, j, self.num_users, self.num_items)
                depth = E.bpr_order_depth(u, i, j, self.num_users, self.num_items)
                E.bpr_sgd_ordered(P, Q, du, di, dj, torch.from_numpy(wu).to(dev), torch.from_numpy(wi).to(dev),
                                  torch.from_numpy(wj).to(dev), self.lRate, self.regU, self.regI, acc[0:1],
                                  n_warps=E.ordered_warps(len(u), depth))
            E.sumsq(P, acc[1:2])
            E.sumsq(Q, acc[2:3])
            a = acc.cpu().numpy()
            self.loss = float(a[0] + self.regU * a[1] + self.regI * a[2])      # BPR.py:40,53
            epoch += 1
            if not self.ranking.isMainOn():
                # isConverged -> rating_performance reads self.P/self.Q (the reference updates them in place)
                self.P = np.ascontiguousarray(P[:, :d].cpu().numpy())
                self.Q = np.ascontiguousarray(Q[:, :d].cpu().numpy())
            if self.isConverged(epoch):
                break
        self.P = np.ascontiguousarray(P[:, :d].cpu().numpy())
        self.Q = np.ascontiguousarray(Q[:, :d].cpu().numpy())

    buildModel = trainModel

    def next_batch(self):
        """(u, i, j) minibatches over trainingData in its current order, negatives from the MT19937
        clone (BPR.py:55-75: like next_batch_pairwise but without the shuffle)."""
        from ... import engine as E
        csr = self.data.rated_csr()
        u_all, i_all, _ = self.data.training_ids()
        mt = E.MT19937()
        for b in range(0, self.train_size, self.batch_size):
            u, i = u_all[b:b + self.batch_size], i_all[b:b + self.batch_size]
            mt.setstate(random.getstate())
            j = mt.sample_pairwise(csr, u)
            random.setstate(mt.getstate())
            yield u, i, j

    def trainModel_tf(self):
        """Minibatch Adam variant (BPR.py:77-96): loss = -sum ln(sigmoid(y)+1e-6)
        + regU*(l2_loss(U)+l2_loss(V)) over the FULL tables; tables start from
        truncated_normal(0.005) (iterativeRecommender.py:44-45)."""
        import torch
        from ... import engine as E
        dev = self._device()
        if not hasattr(self, 'batch_size'):
            self.batch_size = int(self.config['batch_size'])
        d = self.emb_size
        dp = (d + 3) // 4 * 4        # kernels take rows that are a multiple of 4 wide (BPR.conf ships d=50 -> 52);
        U = torch.zeros(self.num_users, dp, device=dev)          # the zero columns stay exactly zero under K3 + Adam
        V = torch.zeros(self.num_items, dp, device=dev)
        U[:, :d] = torch.nn.init.trunc_normal_(torch.empty(self.num_users, d, device=dev), std=0.005, a=-0.01, b=0.01)
        V[:, :d] = torch.nn.init.trunc_normal_(torch.empty(self.num_items, d, device=dev), std=0.005, a=-0.01, b=0.01)
        state = [torch.zeros_like(t) for t in (U, U, V, V)]            # mU, vU, mV, vV
        gU, gV = torch.zeros_like(U), torch.zeros_like(V)
        loss = torch.zeros(3, dtype=torch.float64, device=dev)
        t = 0
        for epoch in range(self.maxEpoch):
            for n, (u, i, j) in enumerate(self.next_batch()):
                t += 1
                # d/dU of regU*l2_loss(U) is regU*U: start the gradient buffers from it
                E.axpby(gU, U, U, self.regU, 0.0)
                E.axpby(gV, V, V, self.regU, 0.0)
                loss.zero_()
                E.bpr_grad_scatter(U, V, torch.from_numpy(u).to(dev), torch.from_numpy(i).to(dev),
                                   torch.from_numpy(j).to(dev), 1e-6, 0.0, gU, gV, loss[0:1])
                E.sumsq(U, loss[1:2]); E.sumsq(V, loss[2:3])
                E.adam_dense_tf1(U, state[0], state[1], gU, self.lRate, t)
                E.adam_dense_tf1(V, state[2], state[3], gV, self.lRate, t)
                if n % 50 == 0:
                    l = loss.cpu().numpy()
                    print('training:', epoch + 1, 'batch', n, 'loss:', l[0] + self.regU * 0.5 * (l[1] + l[2]))
        self.P, self.Q = np.ascontiguousarray(U[:, :d].cpu().numpy()), np.ascontiguousarray(V[:, :d].cpu().numpy())

    def device_tables(self):
        return self._tables_on_device()
