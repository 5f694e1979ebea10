"""Shared trainer of the rating-prediction MF family (BasicMF / PMF / SVD) on the H100 engine.

The reference visits `self.data.trainingData` entry by entry in list order and `isConverged`
reshuffles the list after every epoch (model/rating/PMF.py:13-22, base/iterativeRecommender.py:101).
Here an epoch is one launch over the id-mapped (u, i, r) arrays of the list's current order:
  * engine -mode parity : qrec_mf_sgd_ordered_{f64,f32} -- sequential-equivalent, same tables as the
                          reference after every epoch;
  * engine -mode fast   : one qrec_mf_sgd_batch_f32 launch per epoch over a shuffled list (Hogwild),
                          test pairs scored on the device.  A row hit c times while those hits are
                          in flight moves as if the learning rate were c*lr (every hit reads the same
                          stale row), and the squared-error gradient is unbounded, so the kernel's
                          in-flight window is bounded to (0.25/lr) / (share of the most frequent row)
                          entries: 33 750 user-sorted FilmTrust entries applied as one stale step
                          diverge.
"""
import numpy as np

from ...base.iterativeRecommender import IterativeRecommender


def ordered_rating_pass(model, kind, P, Q, loss, Bu=None, Bi=None):
    """One in-order K9 launch of `kind` over model's training list in its current order: sequential-equivalent, in
    place on the device tables P and Q (and the biases Bu / Bi, around globalMean), with model's learning rate and
    regU / regI / regB.  loss (a float64 slot) += the pass's loss terms."""
    import torch
    from ... import engine as E
    u, i, r = model.data.training_ids()
    wu, wi = E.mf_order_prepare(u, i, model.num_users, model.num_items)
    depth = E.mf_order_depth(u, i, model.num_users, model.num_items)
    t = lambda a: torch.from_numpy(a).to(P.device)                  # noqa: E731
    gm = 0.0 if Bu is None else float(model.data.globalMean)
    E.mf_sgd_ordered(kind, P, Q, t(u), t(i), model._upload(r, P.device), t(wu), t(wi), model.lRate, model.regU,
                     model.regI, loss, Bu, Bi, model.regB, gm, n_warps=E.ordered_warps(len(u), depth))


class PointwiseMF(IterativeRecommender):
    KIND = 1                       # 0 BasicMF, 1 PMF, 2 SVD (include/qrec.h, K9)
    FAST_MAX_INFLIGHT = 1 << 20    # in-flight window of the fast kernel, upper bound (0 would fill the GPU)

    # ------------------------------------------------------------------ reference surface
    def initModel(self):
        super(PointwiseMF, self).initModel()
        self.Bu = self.Bi = None

    def _penalty(self, sums):
        """regulariser of `self.loss` from (|P|^2, |Q|^2, |Bu|^2, |Bi|^2)."""
        return self.regU * sums[0] + self.regI * sums[1]

    # ------------------------------------------------------------------ engine
    def _sync_host_tables(self, P, Q, Bu, Bi):
        self.P, self.Q = self._host(P), self._host(Q)
        if Bu is not None:
            self.Bu, self.Bi = self._host(Bu), self._host(Bi)

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        fast = self.engine_mode == 'fast'
        P, Q = self._upload(self.P, dev, pad=True), self._upload(self.Q, dev, pad=True)
        biased = self.KIND == 2
        Bu = self._upload(self.Bu, dev) if biased else None
        Bi = self._upload(self.Bi, dev) if biased else None
        gm = float(self.data.globalMean) if biased else 0.0
        acc = torch.zeros(5, dtype=torch.float64, device=dev)
        if fast:
            # test pairs are scored from the resident tables
            self._device_scores = lambda tu, ti: E.mf_predict_pairs(P, Q, tu, ti, Bu, Bi, gm)
            u, i, _ = self.data.training_ids()
            top_share = max(int(np.bincount(u).max()), int(np.bincount(i).max())) / float(len(u))
            self.shuffle_training_data()                            # file order is user-sorted: spread the rows
        epoch = 0
        while epoch < self.maxEpoch:
            acc.zero_()
            if fast:
                u, i, r = self.data.training_ids()                  # current (shuffled) list order
                E.mf_sgd_batch(self.KIND, P, Q, torch.from_numpy(u).to(dev), torch.from_numpy(i).to(dev),
                               torch.from_numpy(r).to(device=dev, dtype=P.dtype), self.lRate, self.regU, self.regI,
                               acc[0:1], Bu, Bi, self.regB, gm, max_inflight=self._fast_window(top_share))
            else:
                ordered_rating_pass(self, self.KIND, P, Q, acc[0:1], Bu, Bi)
            if self.KIND != 0:
                E.sumsq(P, acc[1:2]); E.sumsq(Q, acc[2:3])
                if biased:
                    E.sumsq(Bu, acc[3:4]); E.sumsq(Bi, acc[4:5])
            a = acc.cpu().numpy()
            self.loss = float(a[0]) if self.KIND == 0 else float(a[0] + self._penalty(a[1:]))
            if not fast:
                self._sync_host_tables(P, Q, Bu, Bi)                 # rating_performance reads self.P / self.Q
            epoch += 1
            if self._epoch_end(epoch):
                break
        self._sync_host_tables(P, Q, Bu, Bi)
        self._device_scores = None

    buildModel = trainModel

    def _fast_window(self, top_share):
        """In-flight entries of the fast kernel: the most frequent row is hit about 0.25/lr times in it."""
        hits = max(1.0, 0.25 / max(self.lRate, 1e-12))
        return int(min(self.FAST_MAX_INFLIGHT, max(32, hits / max(top_share, 1e-12))))

    def _epoch_end(self, epoch):
        """PMF / BasicMF stop when converged (PMF.py:26-27); SVD ignores the flag (SVD.py:36)."""
        return self.isConverged(epoch)
