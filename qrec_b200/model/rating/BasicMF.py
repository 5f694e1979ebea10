"""BasicMF on the H100 engine -- drop-in for model/rating/BasicMF.py of the reference (kind 0 of K9):
P[u] += lr*e*Q[i]; Q[i] += lr*e*P[u]; loss = sum e^2, no regulariser (BasicMF.py:13-23)."""
from ._pointwise import PointwiseMF


class BasicMF(PointwiseMF):
    KIND = 0

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(BasicMF, self).__init__(conf, trainingSet, testSet, fold)
