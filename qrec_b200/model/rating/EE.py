"""EE on the H100 engine -- drop-in for model/rating/EE.py of the reference (Khoshneshin & Street 2010): a Euclidean
embedding with biases, trained by K9 kind 5 (see _euclidean.py).  `-tf` (the shipped EE.conf sets it) is the base
class's behaviour: a warning, then trainModel."""
from ...base.iterativeRecommender import IterativeRecommender
from ._euclidean import EuclideanMF


class EE(EuclideanMF, IterativeRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(EE, self).__init__(conf, trainingSet, testSet, fold)
