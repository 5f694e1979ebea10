"""Shared pieces of EE and SREE on the H100 engine: the Euclidean-embedding rating model with biases
(model/rating/EE.py, model/rating/SREE.py of the reference).

An epoch is one in-order launch of K9 kind 5 over the training list in its current order (EE.py:18-34):
  dist = |P[u]-Q[i]|^2,  e = r - (((globalMean + Bi[i]) + Bu[u]) - dist),
  P[u] -= (lr*(e+regU))*(P[u]-Q[i]);  Q[i] += (lr*(e+regI))*(P[u](new)-Q[i]);  both biases step from their old values,
followed for SREE by its user pass (K17, SREE.py:48-61).  The loss is sum (e^2 + regU*dist) + regB*|Bu|^2 +
regB*|Bi|^2 (+ SREE's social terms); there is no |P|^2 or |Q|^2 term.  Every maxEpoch epoch runs: isConverged still
adapts the learning rate, reshuffles, prints and stops on NaN, but its verdict is ignored, as in the reference.
Float64 by default, float32 under `engine=-precision f32` or `-mode fast`, on the same in-order kernels.  The host
P, Q, Bu and Bi are refreshed after every epoch, because evaluation and ranking read them.  Ranking adds the distance
(the farthest items rank first), as the reference does, so these models expose no dot-product device_tables() and
`-eval gpu` ranks on the host."""
import numpy as np

from ._pointwise import ordered_rating_pass


class EuclideanMF(object):
    """Mixin ahead of the reference's base class (IterativeRecommender for EE, the social one for SREE)."""

    def initModel(self):
        super(EuclideanMF, self).initModel()
        # two more draws from numpy's global stream, users first (EE.py:11-12, SREE.py:22-23)
        self.Bu = np.random.rand(self.data.trainingSize()[0]) / 10
        self.Bi = np.random.rand(self.data.trainingSize()[1]) / 10

    def _user_pass(self, P):
        """A callable adding the social pass of an epoch to a float64 loss slot, or None (EE)."""
        return None

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        tables = [self._upload(a, dev) for a in (self.P, self.Q, self.Bu, self.Bi)]
        P, Q, Bu, Bi = tables
        user_pass = self._user_pass(P)
        acc = torch.zeros(2, dtype=torch.float64, device=dev)
        epoch = 0
        while epoch < self.maxEpoch:
            acc.zero_()
            ordered_rating_pass(self, E.EE_RATINGS, P, Q, acc[0:1], Bu, Bi)
            if user_pass is not None:
                user_pass(acc[1:2])
            a = acc.cpu().numpy()
            self.P, self.Q, self.Bu, self.Bi = (self._host(x) for x in tables)
            self.loss = float(a[0] + (self.regB * (self.Bu * self.Bu).sum() + self.regB * (self.Bi * self.Bi).sum())
                              + a[1])
            epoch += 1
            self.isConverged(epoch)

    buildModel = trainModel

    def predictForRating(self, u, i):
        if self.data.containsUser(u) and self.data.containsItem(i):
            u, i = self.data.user[u], self.data.item[i]
            return self.data.globalMean + self.Bi[i] + self.Bu[u] - (self.P[u] - self.Q[i]).dot(self.P[u] - self.Q[i])
        return self.data.globalMean

    def predictForRanking(self, u):
        if self.data.containsUser(u):
            u = self.data.user[u]
            return ((self.Q - self.P[u]) * (self.Q - self.P[u])).sum(axis=1) + self.Bi + self.Bu[u] + self.data.globalMean
        return [self.data.globalMean] * self.num_items
