"""The part UserKNN and ItemKNN share (model/rating/UserKNN.py and ItemKNN.py of the reference): neighbour lists and
predictions on the device (K15, engine.knn_neighbours / engine.knn_predict).

Reference behaviour kept as is:
  * `similarity` = pcc / euclidean selects itself, any other value cosine; `num.neighbors` <= 0 reads no neighbour.
  * the candidate list of each test user (item) is the reference's SymmetricMatrix row: every earlier test user
    (cold ones included, with similarity 0) with the similarity the EARLIER one computed, then every other training
    row in id order; it is sorted by similarity descending, stably, so ties keep that order.  The squares are
    CPython's `** 2`, computed on the host (engine.knn_squares), as the reference's bits depend on them.
  * the configuration block, "Computing ... similarities...", a progress line every 100 queries and the completion
    line are printed; the progress lines come after the device call.
  * a prediction whose neighbour sum is 0 returns the query's mean (the global mean for a cold query); a zero
    denominator under a non-zero sum raises ZeroDivisionError.  Item ranking prints the reference's message and exits.
Not kept: the full sorted lists and the SymmetricMatrix of similarities (queries x rows in size).  `topUsers` /
`topItems` hold each query's first `num.neighbors` entries as (name, similarity) pairs.
"""
import sys

import numpy as np

from ...base.recommender import Recommender


class KNNRating(Recommender):
    BY = 'user'            # the side whose rows are compared
    NOUN = 'user'

    def readConfiguration(self):
        super(KNNRating, self).readConfiguration()
        self.sim = self.config['similarity']
        self.neighbors = int(self.config['num.neighbors'])

    def printAlgorConfig(self):
        super(KNNRating, self).printAlgorConfig()
        print('Specified Arguments of', self.config['model.name'] + ':')
        print('num.neighbors:', self.config['num.neighbors'])
        print('similarity:', self.config['similarity'])
        print('=' * 80)

    def _device(self):
        import torch
        return torch.device('cuda')

    # the query side's dicts: (name -> id, id -> name, test queries, means)
    def _side(self):
        d = self.data
        if self.BY == 'user':
            return d.user, d.id2user, d.testSet_u, d.userMeans
        return d.item, d.id2item, d.testSet_i, d.itemMeans

    def initModel(self):
        import torch
        from ... import engine as E
        ids, id2name, queries, means = self._side()
        print('Computing %s similarities...' % self.NOUN)
        rowptr, cols, vals = self.data.rating_csr(self.BY)
        n = len(ids)
        n_cols = len(self.data.item if self.BY == 'user' else self.data.user)
        mean_arr = np.array([means[id2name[k]] for k in range(n)], dtype=np.float64)
        metric = E.knn_metric(self.sim)
        sq = E.knn_squares(rowptr, vals, mean_arr, metric)
        self._query_names = list(queries)
        self._qpos = {name: p for p, name in enumerate(self._query_names)}
        qids = np.array([ids.get(name, -1) for name in self._query_names], dtype=np.int32)
        dev = self._device()
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        self._dev = dict(rowptr=t(rowptr), cols=t(cols), vals=t(vals), means=t(mean_arr), queries=t(qids))
        K = max(self.neighbors, 0)
        nb_ids, nb_sims, nb_cnt = E.knn_neighbours(self._dev['rowptr'], self._dev['cols'], self._dev['vals'], t(sq),
                                                   self._dev['means'], n_cols, self._dev['queries'], metric, K)
        self._dev.update(ids=nb_ids, sims=nb_sims, cnt=nb_cnt)
        self._dev['scols'], self._dev['svals'] = E.knn_sorted_view(self._dev['rowptr'], self._dev['cols'],
                                                                   self._dev['vals'])
        for idx in range(0, len(self._query_names), 100):
            print('progress:', idx, '/', len(self._query_names))
        print('The %s similarities have been calculated.' % self.NOUN)
        ids_h, sims_h, cnt_h = nb_ids.cpu().numpy(), nb_sims.cpu().numpy(), nb_cnt.cpu().numpy()
        top = {}
        for p, name in enumerate(self._query_names):
            row = []
            for k in range(int(cnt_h[p])):
                v = int(ids_h[p, k])
                row.append((id2name[v] if v >= 0 else self._query_names[E.KNN_COLD - v], float(sims_h[p, k])))
            top[name] = row
        self._set_top(top)
        lines = self.data.testData
        self._pred = dict(zip(((r[0], r[1]) for r in lines), zip(*self._predict([r[0] for r in lines],
                                                                               [r[1] for r in lines]))))

    def _set_top(self, top):
        raise NotImplementedError

    def _line(self, u, i):
        """(query name, probe id on the other side) of a test line."""
        raise NotImplementedError

    def _predict(self, users, items):
        import torch
        from ... import engine as E
        qpos, probe = zip(*(self._line(u, i) for u, i in zip(users, items))) if users else ((), ())
        dev = self._dev['cols'].device
        d = self._dev
        pred, status = E.knn_predict(d['rowptr'], d['scols'], d['svals'], d['means'], self.data.globalMean, d['queries'],
                                     d['ids'], d['sims'], d['cnt'], torch.tensor(qpos, dtype=torch.int32, device=dev),
                                     torch.tensor(probe, dtype=torch.int32, device=dev), self.BY == 'user')
        return pred.cpu().numpy().tolist(), status.cpu().numpy().tolist()

    def predictForRating(self, u, i):
        hit = self._pred.get((u, i))
        if hit is None:     # a pair outside the test list: the same kernel on a one-line batch
            hit = tuple(x[0] for x in self._predict([u], [i]))
        pred, status = hit
        if status == 2:
            raise ZeroDivisionError('float division by zero')
        return pred

    def predictForRanking(self, u):
        print('Using Memory based algorithms to rank items is extremely time-consuming. So ranking for all items in '
              '%s is not available.' % self.config['model.name'])
        sys.exit(0)
