"""SoReg on the H100 engine -- drop-in for model/rating/SoReg.py of the reference (Ma et al. 2011).

initModel builds the similarity of every cleaned trust pair (SoReg.py:21-36): for each training user in id order and
each followee f not met yet, Sim[user][f] = Sim[f][user] = (pcc(user, f) + weight(user, f)) / 2.0, the direction met
first fixing both.  The pairs are listed here and their Pearson correlations computed on the device
(engine.knn_pair_similarity, pearson_sp's arithmetic over the training rows).
An epoch is the reference's two passes, each one in-order launch:
  * the rating pass is PMF's step, K9 kind 1 over the training list in its current order (SoReg.py:42-53);
  * the user pass is K17 kind 1 over `social.user` restricted to training users (SoReg.py:54-72):
    P[u] += lr*((-alpha)*(f1 + f2)), f1 / f2 = sum Sim[u][v]*(P[u] - P[v]) over the followees / followers.
The loss is sum e^2 + the reference's running similarity sums + regU|P|^2 + regI|Q|^2, and training stops when
isConverged says so, as in the reference.  P and Q are float64 numpy arrays between epochs."""
from collections import defaultdict

import numpy as np

from ...base.socialRecommender import SocialRecommender
from ...util import config
from ._pointwise import ordered_rating_pass
from ._social_rating import user_pass_setup


class SoReg(SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=list(), fold='[1]'):
        super(SoReg, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(SoReg, self).readConfiguration()
        self.alpha = float(config.OptionConf(self.config['SoReg'])['-alpha'])

    def printAlgorConfig(self):
        super(SoReg, self).printAlgorConfig()
        print('Specified Arguments of', self.config['model.name'] + ':')
        print('alpha: %.3f' % self.alpha)
        print('=' * 80)

    def similarity_pairs(self):
        """The pairs SoReg.py:27-33 computes, in its order: (user names, followee names, a ids, b ids, weights)."""
        seen, xs, ys = set(), [], []
        for user in self.data.user:
            for f in self.social.getFollowees(user):
                if (user, f) not in seen:
                    seen.add((user, f))
                    seen.add((f, user))
                    xs.append(user)
                    ys.append(f)
        a = np.array([self.data.user[x] for x in xs], np.int32)
        b = np.array([self.data.user[y] for y in ys], np.int32)
        w = np.array([self.social.weight(x, y) for x, y in zip(xs, ys)], np.float64)
        return xs, ys, a, b, w

    def initModel(self):
        import torch
        from ... import engine as E
        super(SoReg, self).initModel()
        self.Sim = defaultdict(dict)
        print('constructing similarity matrix...')
        xs, ys, a, b, w = self.similarity_pairs()
        rowptr, cols, vals = self.data.rating_csr('user')
        means = np.array([self.data.userMeans[self.data.id2user[k]] for k in range(len(self.data.user))], np.float64)
        sq = E.knn_squares(rowptr, vals, means, 0)
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(self._device())   # noqa: E731
        drow, dcols = t(rowptr), t(cols)
        scols, svals = E.knn_sorted_view(drow, dcols, t(vals))
        _, ssq = E.knn_sorted_view(drow, dcols, t(sq))
        sims = E.knn_pair_similarity(drow, dcols, t(vals), t(sq), t(means), scols, svals, ssq, t(a), t(b),
                                     t(w)).cpu().numpy().tolist()
        for x, y, s in zip(xs, ys, sims):
            self.Sim[x][y] = s
            self.Sim[y][x] = s

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        P, Q = self._upload(self.P, dev), self._upload(self.Q, dev)
        social, sim_g, pass_warps = user_pass_setup(self, P, self.Sim)
        acc = torch.zeros(4, dtype=torch.float64, device=dev)
        epoch = 0
        while epoch < self.maxEpoch:
            acc.zero_()
            ordered_rating_pass(self, 1, P, Q, acc[0:1])
            E.social_user_pass(E.SOCIAL_PASS_KINDS['SoReg'], P, *social, sim_g, self.lRate, self.alpha, acc[1:2],
                               n_warps=pass_warps)
            E.sumsq(P, acc[2:3]); E.sumsq(Q, acc[3:4])
            a = acc.cpu().numpy()
            self.loss = float(a[0] + a[1] + (self.regU * a[2] + self.regI * a[3]))
            self.P, self.Q = self._host(P), self._host(Q)
            epoch += 1
            if self.isConverged(epoch):
                break

    buildModel = trainModel
