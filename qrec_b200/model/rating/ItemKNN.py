"""ItemKNN on the H100 engine -- drop-in for model/rating/ItemKNN.py of the reference.  The neighbour lists of every
test item and the predictions of every test line are computed on the device (engine.knn_neighbours, K15); see
_knn.py for the reference behaviour kept.  A neighbour item n counts when `contains(u, n)`, whatever the stored
rating.  `topItems[i]` holds i's first `num.neighbors` (name, similarity) pairs; the reference's full sorted lists and
its `itemSim` matrix are not kept (test items x items in size)."""
from ._knn import KNNRating


class ItemKNN(KNNRating):
    BY = 'item'
    NOUN = 'item'

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(ItemKNN, self).__init__(conf, trainingSet, testSet, fold)

    def _set_top(self, top):
        self.topItems = top

    def _line(self, u, i):
        return self._qpos[i], self.data.user.get(u, -1)
