"""RSTE on the H100 engine -- drop-in for model/rating/RSTE.py of the reference (Ma et al. 2009).

Each training entry (u, i) predicts from u's own row and from the rows of u's followees,
    alpha*(P[u].Q[i]) + ((1-alpha)*sum_f w_f (P[f].Q[i])) / denom[u]    (P[u].Q[i] alone when denom[u] == 0),
and updates P[u] and Q[i] with PMF's step on the error alpha*e (RSTE.py:20-64).  An epoch is one in-order launch
of K16 (qrec_rste_sgd_ordered_*) over the training list in its current order; the loss is sum e^2 + regU|P|^2 +
regI|Q|^2.  Training runs every epoch: isConverged's verdict is ignored, but it still adapts the learning rate and
shuffles the list, as in the reference.  The per-epoch test evaluation scores the known pairs on the device
(qrec_rste_predict_pairs_*).  P and Q are float64 numpy arrays between epochs."""
import numpy as np

from ...base.socialRecommender import SocialRecommender
from ...util import config
from ._social_rating import followee_csr


class RSTE(SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=list(), fold='[1]'):
        super(RSTE, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(RSTE, self).readConfiguration()
        self.alpha = float(config.OptionConf(self.config['RSTE'])['-alpha'])

    def printAlgorConfig(self):
        super(RSTE, self).printAlgorConfig()
        print('Specified Arguments of', self.config['model.name'] + ':')
        print('alpha: %.3f' % self.alpha)
        print('=' * 80)

    def _followees(self):
        if not hasattr(self, '_csr'):
            self._csr = followee_csr(self.data, self.social)
        return self._csr

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        U = self.num_users
        P, Q = self._upload(self.P, dev), self._upload(self.Q, dev)
        rowptr, cols, w, denom = self._followees()
        social = (torch.from_numpy(rowptr).to(dev), torch.from_numpy(cols).to(dev), self._upload(w, dev),
                  self._upload(denom, dev))
        acc = torch.zeros(3, dtype=torch.float64, device=dev)
        # the per-epoch test evaluation scores the known pairs from the resident tables
        self._device_scores = lambda tu, ti: E.rste_predict_pairs(P, Q, tu, ti, *social, self.alpha)
        epoch = 0
        while epoch < self.maxEpoch:
            u, i, r = self.data.training_ids()                     # current (shuffled) list order
            wu, wi, wr, pos_rowptr, pos, depth = E.rste_order_prepare(u, i, U, self.num_items, rowptr, cols)
            dv = [torch.from_numpy(a).to(dev) for a in (u, i, wu, wi, wr, pos_rowptr, pos)]
            acc.zero_()
            E.rste_sgd_ordered(P, Q, dv[0], dv[1], self._upload(r, dev), dv[2], dv[3], dv[4], dv[5], dv[6], *social,
                               self.lRate, self.regU, self.regI, self.alpha, acc[0:1],
                               n_warps=E.ordered_warps(len(u), depth))
            E.sumsq(P, acc[1:2]); E.sumsq(Q, acc[2:3])
            a = acc.cpu().numpy()
            self.loss = float(a[0] + (self.regU * a[1] + self.regI * a[2]))
            self.P, self.Q = self._host(P), self._host(Q)
            epoch += 1
            self.isConverged(epoch)                                # RSTE.py:39: the verdict is not used
        self._device_scores = None

    buildModel = trainModel

    def predictForRating(self, u, i):
        """RSTE.py:41-64 on the host tables, for the final evaluation and single pairs."""
        if not (self.data.containsUser(u) and self.data.containsItem(i)):
            return self.data.globalMean
        uid, iid = self.data.user[u], self.data.getItemId(i)
        cols, w, denom = self._followee_arrays(uid)
        if denom != 0:
            social = 0
            social += w.dot(self.P[cols].dot(self.Q[iid]))
            return self.alpha * self.P[uid].dot(self.Q[iid]) + (1 - self.alpha) * social / denom
        return self.P[uid].dot(self.Q[iid])

    def _followee_arrays(self, uid):
        """u's followee ids and weights as the reference's numpy arrays, and their sum."""
        name = self.data.id2user[uid]
        ids, weights = [], []
        for f, wf in self.social.getFollowees(name).items():
            if self.data.containsUser(f):
                ids.append(self.data.user[f])
                weights.append(wf)
        weights = np.array(weights)
        return np.array(ids), weights, weights.sum()

    def predictForRanking(self, u):
        """RSTE.py:66-83: the blend over all items, with the followee terms summed row by row in Python."""
        if not self.data.containsUser(u):
            return [self.data.globalMean] * len(self.data.item)
        social, total = 0, 0
        for f, wf in self.social.getFollowees(u).items():
            if self.data.containsUser(f):
                social += wf * self.Q.dot(self.P[self.data.user[f]])
                total += wf
        own = self.Q.dot(self.P[self.data.user[u]])
        if total != 0:
            return self.alpha * own + (1 - self.alpha) * social / total
        return own
