"""PMF on the H100 engine -- drop-in for model/rating/PMF.py of the reference (kind 1 of K9):
P[u] += lr*(e*Q[i] - regU*P[u]); Q[i] += lr*(e*P[u] - regI*Q[i]); loss = sum e^2 + regU|P|^2 + regI|Q|^2
(PMF.py:13-24)."""
from ._pointwise import PointwiseMF


class PMF(PointwiseMF):
    KIND = 1

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(PMF, self).__init__(conf, trainingSet, testSet, fold)
