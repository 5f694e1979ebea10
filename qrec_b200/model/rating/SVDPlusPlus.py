"""SVD++ on the H100 engine -- drop-in for model/rating/SVDPlusPlus.py of the reference (K11).

The model adds an implicit-factor table Y[num_items, d]: an entry (u, i, r) predicts with the mean of the Y rows of
every item the user rated and then updates all of those rows but Y[i] (SVDPlusPlus.py:26-88).  Every entry depends
on almost every entry before it, so there are two engines:
  * -mode parity (default): qrec_svdpp_sgd_ordered_{f64,f32} -- the entries of `trainingData` in its current list
    order, one after another on one CTA, in the reference's evaluation order.  float64 tables (float32 with
    `-precision f32`); the host tables are refreshed every epoch for rating_performance.
  * -mode fast: qrec_svdpp_epoch_usermajor_f32 -- one user-major epoch per launch, users longest first, each user's
    entries through the per-user closed form (csrc/svdpp_step.cuh).  fp32 tables padded to a multiple of 4 columns;
    test pairs are scored on the device.  It runs on the de-duplicated user CSR (`rating_csr('user')`): a repeated
    (user, item) line is one entry with the line's last value, where the reference visits every line.  Users in
    flight read each other's item rows stale, so at most (0.25/lr) / (share of the users who rated the most-rated
    item) users run at a time.

Reference behaviour kept as is:
  * the prediction divides the sum of all w rows of N(u) by w, while the Q step sums the w-1 rows j != i;
  * there is no |N(u)|^-1/2 normalisation (Koren's form is not used);
  * Bu, Bi, Y are drawn with np.random.rand after P and Q, without SVD's /5;
  * every epoch runs: isConverged (which reshuffles trainingData and scores the test set) never stops training;
  * predictForRanking exists, although SVD++.conf ranks nothing.
"""
import numpy as np

from ._pointwise import PointwiseMF
from ...util.config import OptionConf


class SVDPlusPlus(PointwiseMF):
    KIND = None                    # not a K9 kind: trains with K11

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(SVDPlusPlus, self).__init__(conf, trainingSet, testSet, fold)

    def readConfiguration(self):
        super(SVDPlusPlus, self).readConfiguration()
        regY = OptionConf(self.config['SVDPlusPlus'])
        self.regY = float(regY['-y'])

    def printAlgorConfig(self):
        super(SVDPlusPlus, self).printAlgorConfig()
        print('Specified Arguments of', self.config['model.name'] + ':')
        print('regY: %.3f' % self.regY)
        print('=' * 80)

    def initModel(self):
        super(SVDPlusPlus, self).initModel()
        # three more draws from numpy's global stream, in this order (SVDPlusPlus.py:22-24)
        self.Bu = np.random.rand(self.data.trainingSize()[0])
        self.Bi = np.random.rand(self.data.trainingSize()[1])
        self.Y = np.random.rand(self.data.trainingSize()[1], self.emb_size)

    # ------------------------------------------------------------------ engine
    def _users_in_flight(self, top_share):
        """Users of the fast epoch at a time: the most-rated item is then visited about 0.25/lr times in flight."""
        hits = max(1.0, 0.25 / max(self.lRate, 1e-12))
        return int(min(self.FAST_MAX_INFLIGHT, max(1, hits / max(top_share, 1e-12))))

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        fast = self.engine_mode == 'fast'
        P, Q, Y = (self._upload(t, dev, pad=True) for t in (self.P, self.Q, self.Y))
        Bu, Bi = self._upload(self.Bu, dev), self._upload(self.Bi, dev)
        gm = float(self.data.globalMean)
        rowptr, cols, vals = self.data.rating_csr('user')
        drp, dcols = torch.from_numpy(rowptr).to(dev), torch.from_numpy(cols).to(dev)
        acc = torch.zeros(6, dtype=torch.float64, device=dev)
        if fast:
            dvals = torch.from_numpy(vals).to(device=dev, dtype=P.dtype)
            order = torch.from_numpy(E.als_row_order(rowptr)).to(dev)
            top_share = np.bincount(cols, minlength=self.num_items).max() / float(max(1, self.num_users))
            ivals = torch.from_numpy(1.0 / np.repeat(np.diff(rowptr), np.diff(rowptr))).to(device=dev, dtype=P.dtype)

            def scores(tu, ti):
                """Test pairs scored from the resident tables: Z = D^-1 R Y (the mean implicit row of every user,
                qrec_spmm_csr_f32 with values 1/w), then Z[u].Q[i] + (P[u].Q[i] + mean + Bi[i] + Bu[u])."""
                Z = torch.empty_like(P)
                E.spmm_csr(drp, dcols, ivals, Y, Z)
                return E.mf_predict_pairs(Z, Q, tu, ti).double() + E.mf_predict_pairs(P, Q, tu, ti, Bu, Bi, gm).double()
            self._device_scores = scores
        epoch = 0
        while epoch < self.maxEpoch:
            acc.zero_()
            if fast:
                E.svdpp_epoch_usermajor(P, Q, Y, Bu, Bi, drp, dcols, dvals, order, self.lRate, self.regU, self.regI,
                                        self.regB, self.regY, gm, acc[0:1],
                                        max_users_in_flight=self._users_in_flight(top_share))
            else:
                u, i, r = self.data.training_ids()                  # current (shuffled) list order
                E.svdpp_sgd_ordered(P, Q, Y, Bu, Bi, torch.from_numpy(u).to(dev), torch.from_numpy(i).to(dev),
                                    torch.from_numpy(r).to(device=dev, dtype=P.dtype), drp, dcols, self.lRate,
                                    self.regU, self.regI, self.regB, self.regY, gm, acc[0:1])
            for k, t in enumerate((P, Q, Y, Bu, Bi)):
                E.sumsq(t, acc[k + 1:k + 2])
            a = acc.cpu().numpy()
            self.loss = float(a[0] + (self.regU * a[1] + self.regI * a[2] + self.regY * a[3]
                                      + self.regB * (a[4] + a[5])))
            if not fast:
                self.Y = self._host(Y)                              # rating_performance reads the host tables
                self._sync_host_tables(P, Q, Bu, Bi)
            epoch += 1
            self.isConverged(epoch)                                 # SVDPlusPlus.py:67: never stops training
        self.Y = self._host(Y)
        self._sync_host_tables(P, Q, Bu, Bi)
        self._device_scores = None

    buildModel = trainModel

    def predictForRating(self, u, i):
        """SVDPlusPlus.py:70-88, in its order: sequential row sum, /w, dot, then P.Q + mean + Bi + Bu."""
        pred = 0
        if self.data.containsUser(u) and self.data.containsItem(i):
            itemIndexs, _ = self.data.userRated(u)
            w = len(itemIndexs)
            u, i = self.data.user[u], self.data.item[i]
            s = 0
            if w > 0:
                for j in itemIndexs:
                    s += self.Y[self.data.item[j]]
                pred += (s / w).dot(self.Q[i])
            pred += self.P[u].dot(self.Q[i]) + self.data.globalMean + self.Bi[i] + self.Bu[u]
        else:
            pred = self.data.globalMean
        return pred

    def predictForRanking(self, u):
        """SVDPlusPlus.py:90-107"""
        pred = 0
        if self.data.containsUser(u):
            itemIndexs, _ = self.data.userRated(u)
            w = len(itemIndexs)
            u = self.data.user[u]
            s = 0
            if w > 0:
                for j in itemIndexs:
                    s += self.Y[self.data.item[j]]
                pred += self.Q.dot(s / w)
            pred += self.Q.dot(self.P[u]) + self.data.globalMean + self.Bi + self.Bu[u]
        else:
            pred = [self.data.globalMean] * self.num_items
        return pred
