"""`Rating`: the id space and per-user / per-item views of the training and test sets.

Same public attributes and id assignment as the reference (data/rating.py:5-190): users and items
receive dense ids in order of first appearance in the training list; `trainSet_u[user][item]`
holds the rating (a repeated (user,item) line overwrites the value but keeps its position).
On top of the dict views this class keeps the id-mapped training list as int32 arrays
(`train_u_ids`, `train_i_ids`) and hands the engine a `RatedCSR` -- that is what the kernels and
the C samplers consume.
"""
import random
from collections import defaultdict

import numpy as np

from ..util.config import OptionConf


class Rating(object):
    def __init__(self, config, trainingSet, testSet):
        self.config = config
        self.evalSettings = OptionConf(self.config['evaluation.setup'])
        self.user, self.item = {}, {}
        self.id2user, self.id2item = {}, {}
        self.userMeans, self.itemMeans = {}, {}
        self.globalMean = 0
        self.trainSet_u, self.trainSet_i = defaultdict(dict), defaultdict(dict)
        self.testSet_u, self.testSet_i = defaultdict(dict), defaultdict(dict)
        self.rScale = []
        self.trainingData = trainingSet[:]
        self.testData = testSet[:]
        self._csr = None
        self._index_training_set()
        self._index_test_set()
        self._means()
        if self.evalSettings.contains('-cold'):
            self._keep_cold_start_users(int(self.evalSettings['-cold']))

    # ------------------------------------------------------------------ construction
    def _index_training_set(self):
        if self.evalSettings.contains('-val'):
            # validation split carved out of the training list (consumes the global MT19937)
            random.shuffle(self.trainingData)
            cut = int(self.elemCount() * float(self.evalSettings['-val']))
            self.testData = self.trainingData[:cut]
            self.trainingData = self.trainingData[cut:]
        seen = set()
        users, items = self.user, self.item
        for name_u, name_i, value in self.trainingData:
            if name_u not in users:
                users[name_u] = len(users)
                self.id2user[users[name_u]] = name_u
            if name_i not in items:
                items[name_i] = len(items)
                self.id2item[items[name_i]] = name_i
            self.trainSet_u[name_u][name_i] = value
            self.trainSet_i[name_i][name_u] = value
            seen.add(float(value))
        self.rScale = sorted(seen)

    def _index_test_set(self):
        if self.evalSettings.contains('-predict'):
            for name_u in self.testData:
                self.testSet_u[name_u] = {}
            return
        for name_u, name_i, value in self.testData:
            self.testSet_u[name_u][name_i] = value
            self.testSet_i[name_i][name_u] = value

    def _means(self):
        for name_u in self.user:
            row = self.trainSet_u[name_u]
            self.userMeans[name_u] = sum(row.values()) / len(row)
        for name_i in self.item:
            col = self.trainSet_i[name_i]
            self.itemMeans[name_i] = sum(col.values()) / len(col)
        total = sum(self.userMeans.values())
        self.globalMean = total / len(self.userMeans) if total != 0 else 0

    def _keep_cold_start_users(self, threshold):
        warm = {u for u in self.testSet_u if u in self.trainSet_u and len(self.trainSet_u[u]) > threshold}
        for u in warm:
            del self.testSet_u[u]
        self.testData = [rec for rec in self.testData if rec[0] not in warm]

    # ------------------------------------------------------------------ engine views
    def training_ids(self):
        """(u_ids, i_ids, ratings) of `trainingData` in its CURRENT order, int32/int32/float64."""
        n = len(self.trainingData)
        u = np.fromiter((self.user[r[0]] for r in self.trainingData), dtype=np.int32, count=n)
        i = np.fromiter((self.item[r[1]] for r in self.trainingData), dtype=np.int32, count=n)
        r = np.fromiter((r[2] for r in self.trainingData), dtype=np.float64, count=n)
        return u, i, r

    def rated_csr(self):
        """RatedCSR of trainSet_u: positives in insertion order + all rated items sorted."""
        if self._csr is None:
            from ..engine import RatedCSR
            u = np.empty(0, np.int64); i = np.empty(0, np.int64); r = np.empty(0, np.float64)
            rows = [(self.user[name_u], self.item[name_i], val)
                    for name_u, row in self.trainSet_u.items() if name_u in self.user
                    for name_i, val in row.items()]
            if rows:
                arr = np.array(rows, dtype=np.float64)
                u, i, r = arr[:, 0].astype(np.int64), arr[:, 1].astype(np.int64), arr[:, 2]
            self._csr = RatedCSR(len(self.user), len(self.item), u, i, r)
        return self._csr

    def rating_csr(self, by='user'):
        """(rowptr int64, cols int32, vals float64) of trainSet_u (by='user': rows are user ids, columns item ids)
        or trainSet_i (by='item': rows are item ids, columns user ids), each row in the dict's insertion order.
        Built from the dicts, so a repeated (user, item) line counts once with its last value and `-b` is already
        applied -- the entries WRMF.py:30-36 / 51-57 visit."""
        if by not in ('user', 'item'):
            raise ValueError("by must be 'user' or 'item'")
        cache = self.__dict__.setdefault('_rating_csr', {})
        if by not in cache:
            rows, names, ids, other = ((self.trainSet_u, self.id2user, self.user, self.item) if by == 'user'
                                       else (self.trainSet_i, self.id2item, self.item, self.user))
            lengths = np.fromiter((len(rows[names[k]]) for k in range(len(ids))), dtype=np.int64, count=len(ids))
            rowptr = np.zeros(len(ids) + 1, dtype=np.int64)
            np.cumsum(lengths, out=rowptr[1:])
            n = int(rowptr[-1])
            cols = np.fromiter((other[c] for k in range(len(ids)) for c in rows[names[k]]), dtype=np.int32, count=n)
            vals = np.fromiter((float(v) for k in range(len(ids)) for v in rows[names[k]].values()), dtype=np.float64,
                               count=n)
            cache[by] = (rowptr, cols, vals)
        return cache[by]

    # ------------------------------------------------------------------ reference API
    def getUserId(self, u):
        return self.user.get(u)

    def getItemId(self, i):
        return self.item.get(i)

    def trainingSize(self):
        return (len(self.user), len(self.item), len(self.trainingData))

    def testSize(self):
        return (len(self.testSet_u), len(self.testSet_i), len(self.testData))

    def contains(self, u, i):
        return u in self.user and i in self.trainSet_u[u]

    def containsUser(self, u):
        return u in self.user

    def containsItem(self, i):
        return i in self.item

    def userRated(self, u):
        row = self.trainSet_u[u]
        return list(row.keys()), list(row.values())

    def itemRated(self, i):
        col = self.trainSet_i[i]
        return list(col.keys()), list(col.values())

    def row(self, u):
        vec = np.zeros(len(self.item))
        for name_i, val in self.trainSet_u[u].items():
            vec[self.item[name_i]] = val
        return vec

    def col(self, i):
        vec = np.zeros(len(self.user))
        for name_u, val in self.trainSet_i[i].items():
            vec[self.user[name_u]] = val
        return vec

    def matrix(self):
        m = np.zeros((len(self.user), len(self.item)))
        for name_u, uid in self.user.items():
            m[uid] = self.row(name_u)
        return m

    def sRow(self, u):
        return self.trainSet_u[u]

    def sCol(self, c):
        return self.trainSet_i[c]

    def rating(self, u, c):
        return self.trainSet_u[u][c] if self.contains(u, c) else -1

    def ratingScale(self):
        return (self.rScale[0], self.rScale[1])

    def elemCount(self):
        return len(self.trainingData)
