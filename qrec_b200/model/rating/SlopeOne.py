"""SlopeOne on the H100 engine -- drop-in for model/rating/SlopeOne.py of the reference.

initModel computes the prediction of every test line in one launch (engine.slopeone_predict, K15): for each test item
the kernel builds its diff / count row against every training item (the item itself included) from the item's users
in insertion order, and serves the item's test lines from it.

Reference behaviour kept as is:
  * diff sums x_i[u] - x_j[u] over i's users in trainSet_i order that also rated j; the stored average is diff/count,
    or 0 with count 0.
  * a warm user's prediction walks the user's rated items in insertion order: sum((r + diff) * count) / sum(count),
    the user's mean when the counts sum to 0; a cold user gets the item's mean, or the global mean for a cold item.
  * the "item ... finished." line of every test item is printed (after the device call).
Not kept: the `diffAverage` and `freq` dicts (test items x items in size).  A pair outside the test list goes
through the same kernel as a one-line batch.
"""
import numpy as np

from ...base.recommender import Recommender


class SlopeOne(Recommender):
    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(SlopeOne, self).__init__(conf, trainingSet, testSet, fold)

    def _device(self):
        import torch
        return torch.device('cuda')

    def initModel(self):
        import torch
        d = self.data
        dev = self._device()
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        irp, icols, ivals = d.rating_csr('item')
        urp, ucols, uvals = d.rating_csr('user')
        self._test_items = list(d.testSet_i)
        self._qpos = {name: p for p, name in enumerate(self._test_items)}
        self._dev = dict(
            irp=t(irp), icols=t(icols), ivals=t(ivals),
            imeans=t(np.array([d.itemMeans[d.id2item[k]] for k in range(len(d.item))], dtype=np.float64)),
            urp=t(urp), ucols=t(ucols), uvals=t(uvals),
            umeans=t(np.array([d.userMeans[d.id2user[k]] for k in range(len(d.user))], dtype=np.float64)),
            items=t(np.array([d.item.get(name, -1) for name in self._test_items], dtype=np.int32)))
        lines = d.testData
        users, items = [r[0] for r in lines], [r[1] for r in lines]
        self._pred = dict(zip(zip(users, items), self._predict(users, items)))
        for name in self._test_items:
            print('item ' + name + " finished.")

    def _predict(self, users, items):
        import torch
        from ... import engine as E
        dv = self._dev
        dev = dv['icols'].device
        qpos = torch.tensor([self._qpos[i] for i in items], dtype=torch.int32, device=dev)
        uid = torch.tensor([self.data.user.get(u, -1) for u in users], dtype=torch.int32, device=dev)
        pred, _ = E.slopeone_predict(dv['irp'], dv['icols'], dv['ivals'], dv['imeans'], dv['urp'], dv['ucols'],
                                     dv['uvals'], dv['umeans'], self.data.globalMean, dv['items'], qpos, uid)
        return pred.cpu().numpy().tolist()

    def predictForRating(self, u, i):
        pred = self._pred.get((u, i))
        return self._predict([u], [i])[0] if pred is None else pred
