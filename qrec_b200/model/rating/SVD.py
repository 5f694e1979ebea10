"""SVD (biased MF) on the H100 engine -- drop-in for model/rating/SVD.py of the reference (kind 2 of
K9): PMF's step with e taken against P[u].Q[i] + globalMean + Bi[i] + Bu[u], plus the two bias
updates and their regB penalty (SVD.py:17-34); training runs all epochs (SVD.py:36 ignores the
convergence flag)."""
import numpy as np

from ._pointwise import PointwiseMF


class SVD(PointwiseMF):
    KIND = 2

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(SVD, self).__init__(conf, trainingSet, testSet, fold)

    def initModel(self):
        super(SVD, self).initModel()
        # two more draws from numpy's global stream, users first (SVD.py:11-12)
        self.Bu = np.random.rand(self.data.trainingSize()[0]) / 5
        self.Bi = np.random.rand(self.data.trainingSize()[1]) / 5

    def _penalty(self, sums):
        return self.regU * sums[0] + self.regI * sums[1] + self.regB * (sums[2] + sums[3])

    def _epoch_end(self, epoch):
        self.isConverged(epoch)
        return False

    def predictForRating(self, u, i):
        if self.data.containsUser(u) and self.data.containsItem(i):
            u, i = self.data.user[u], self.data.item[i]
            return self.P[u].dot(self.Q[i]) + self.data.globalMean + self.Bi[i] + self.Bu[u]
        return self.data.globalMean

    def predictForRanking(self, u):
        if self.data.containsUser(u):
            u = self.data.getUserId(u)
            return self.Q.dot(self.P[u]) + self.data.globalMean + self.Bi + self.Bu[u]
        return [self.data.globalMean] * self.num_items
