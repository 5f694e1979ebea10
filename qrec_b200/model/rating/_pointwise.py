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
from ...util.measure import Measure


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
    def _upload(self, a, dev, dtype, dpad=None):
        import torch
        if a.ndim == 1:
            return torch.from_numpy(a).to(device=dev, dtype=dtype).contiguous()
        t = torch.zeros(a.shape[0], dpad, device=dev, dtype=dtype)
        t[:, :a.shape[1]] = torch.from_numpy(a).to(device=dev, dtype=dtype)
        return t.contiguous()

    def _sync_host_tables(self, P, Q, Bu, Bi):
        d = self.emb_size
        self.P = np.ascontiguousarray(P[:, :d].double().cpu().numpy())
        self.Q = np.ascontiguousarray(Q[:, :d].double().cpu().numpy())
        if Bu is not None:
            self.Bu, self.Bi = Bu.double().cpu().numpy(), Bi.double().cpu().numpy()

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        fast = self.engine_mode == 'fast'
        dtype = torch.float32 if (fast or self.engine_precision == 'f32') else torch.float64
        d = self.emb_size
        dpad = d if (not fast or d % 4 == 0) else d + (4 - d % 4)      # zero columns stay zero under the update
        P, Q = self._upload(self.P, dev, dtype, dpad), self._upload(self.Q, dev, dtype, dpad)
        biased = self.KIND == 2
        Bu = self._upload(self.Bu, dev, dtype) if biased else None
        Bi = self._upload(self.Bi, dev, dtype) if biased else None
        gm = float(self.data.globalMean) if biased else 0.0
        acc = torch.zeros(5, dtype=torch.float64, device=dev)
        self._device_state = (P, Q, Bu, Bi, gm) if fast else None
        top_share = 1.0
        if fast:
            u, i, _ = self.data.training_ids()
            top_share = max(int(np.bincount(u).max()), int(np.bincount(i).max())) / float(len(u))
            self.shuffle_training_data()                            # file order is user-sorted: spread the rows
        epoch = 0
        while epoch < self.maxEpoch:
            u, i, r = self.data.training_ids()                      # current (shuffled) list order
            window = self._fast_window(top_share)
            du, di = torch.from_numpy(u).to(dev), torch.from_numpy(i).to(dev)
            dr = torch.from_numpy(r).to(device=dev, dtype=dtype)
            acc.zero_()
            if fast:
                E.mf_sgd_batch(self.KIND, P, Q, du, di, dr, self.lRate, self.regU, self.regI, acc[0:1], Bu, Bi,
                               self.regB, gm, max_inflight=window)
            else:
                wu, wi = E.mf_order_prepare(u, i, self.num_users, self.num_items)
                width = len(u) / max(1, E.mf_order_depth(u, i, self.num_users, self.num_items))
                E.mf_sgd_ordered(self.KIND, P, Q, du, di, dr, torch.from_numpy(wu).to(dev), torch.from_numpy(wi).to(dev),
                                 self.lRate, self.regU, self.regI, acc[0:1], Bu, Bi, self.regB, gm,
                                 n_warps=int(min(2368, max(64, 16 * width))))
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
        self._device_state = None

    buildModel = trainModel

    def _fast_window(self, top_share):
        """In-flight entries of the fast kernel: the most frequent row is hit about 0.25/lr times in it."""
        hits = max(1.0, 0.25 / max(self.lRate, 1e-12))
        return int(min(self.FAST_MAX_INFLIGHT, max(32, hits / max(top_share, 1e-12))))

    def _epoch_end(self, epoch):
        """PMF / BasicMF stop when converged (PMF.py:26-27); SVD ignores the flag (SVD.py:36)."""
        return self.isConverged(epoch)

    # ------------------------------------------------------------------ evaluation
    def rating_performance(self):
        """iterativeRecommender.py:104-113.  In fast mode the known (user, item) pairs of the test set are
        scored on the device from the resident tables; unknown users / items fall back to the means as
        in predictForRating (iterativeRecommender.py:66-73)."""
        state = getattr(self, '_device_state', None)
        if state is None:
            return super(PointwiseMF, self).rating_performance()
        import torch
        from ... import engine as E
        P, Q, Bu, Bi, gm = state
        if not hasattr(self, '_test_pairs'):
            known = [k for k, (un, it, _) in enumerate(self.data.testData)
                     if self.data.containsUser(un) and self.data.containsItem(it)]
            tu = np.array([self.data.user[self.data.testData[k][0]] for k in known], dtype=np.int32)
            ti = np.array([self.data.item[self.data.testData[k][1]] for k in known], dtype=np.int32)
            self._test_pairs = (known, torch.from_numpy(tu).to(P.device), torch.from_numpy(ti).to(P.device))
        known, tu, ti = self._test_pairs
        scores = E.mf_predict_pairs(P, Q, tu, ti, Bu, Bi, gm).double().cpu().numpy()
        res, pos = [], dict(zip(known, range(len(known))))
        for k, (user, item, rating) in enumerate(self.data.testData):
            pred = float(scores[pos[k]]) if k in pos else self.predictForRating(user, item)
            res.append([user, item, rating, self.checkRatingBoundary(pred)])
        self.measure = Measure.ratingMeasure(res)
        return self.measure
