"""UserKNN on the H100 engine -- drop-in for model/rating/UserKNN.py of the reference.  The neighbour lists of every
test user and the predictions of every test line are computed on the device (engine.knn_neighbours, K15); see
_knn.py for the reference behaviour kept.  A neighbour counts for item i when `rating(n, i) != -1`, so a stored rating
of exactly -1 is skipped.  `topUsers[u]` holds u's first `num.neighbors` (name, similarity) pairs; the reference's
full sorted lists and its `userSim` matrix are not kept (test users x users in size)."""
from ._knn import KNNRating


class UserKNN(KNNRating):
    BY = 'user'
    NOUN = 'user'

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(UserKNN, self).__init__(conf, trainingSet, testSet, fold)

    def _set_top(self, top):
        self.topUsers = top

    def _line(self, u, i):
        return self._qpos[u], self.data.item.get(i, -1)
