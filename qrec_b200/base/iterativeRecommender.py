"""`IterativeRecommender`: hyper-parameters, the float64 P/Q tables of the numpy-style models, the
adaptive learning rate and the convergence test (reference: base/iterativeRecommender.py:13-185).

Engine options (not in the reference) come from an optional `engine=` line of the .conf file:
    engine=-mode parity|fast -precision f64|f32 -device 0 -seed 0
`parity` (default) reproduces the reference's sequential SGD exactly; `fast` is the fused
throughput kernel.  Everything else is read from the same keys as the reference.
"""
import random
import sys
from math import isnan

import numpy as np

from .recommender import Recommender
from ..util.config import OptionConf
from ..util.measure import Measure
from ..util.qmath import find_k_largest


class IterativeRecommender(Recommender):
    score_tables = ('P', 'Q')          # the (user, item) tables with score(u, i) = U[u] . V[i]

    def __init__(self, conf, trainingSet, testSet, fold='[1]'):
        super(IterativeRecommender, self).__init__(conf, trainingSet, testSet, fold)
        self.bestPerformance = []
        self.earlyStop = 0
        self._device_scores = None

    def readConfiguration(self):
        super(IterativeRecommender, self).readConfiguration()
        self.emb_size = int(self.config['num.factors'])
        self.maxEpoch = int(self.config['num.max.epoch'])
        rate = OptionConf(self.config['learnRate'])
        self.lRate = float(rate['-init'])
        self.maxLRate = float(rate['-max'])
        if self.evalSettings.contains('-tf'):
            self.batch_size = int(self.config['batch_size'])
        reg = OptionConf(self.config['reg.lambda'])
        self.regU, self.regI, self.regB = float(reg['-u']), float(reg['-i']), float(reg['-b'])
        eng = OptionConf(self.config['engine']) if self.config.contains('engine') else None
        self.engine_mode = eng['-mode'] if eng and eng.contains('-mode') else 'parity'
        self.engine_precision = eng['-precision'] if eng and eng.contains('-precision') else 'f64'
        self.engine_device = int(eng['-device']) if eng and eng.contains('-device') else 0
        self.engine_seed = int(eng['-seed']) if eng and eng.contains('-seed') else 0
        if self.engine_mode not in ('parity', 'fast') or self.engine_precision not in ('f64', 'f32'):
            print('engine option is invalid! use -mode parity|fast -precision f64|f32')
            sys.exit(-1)

    def _device(self):
        """The CUDA device named by `engine=-device N` (made current); the one place the numpy-style
        models touch torch.cuda, so that host-logic tests can swap it."""
        import torch
        dev = torch.device('cuda', self.engine_device)
        torch.cuda.set_device(dev)
        return dev

    def _engine_dtype(self):
        """The dtype of the device tables: float32 under `-mode fast` or `-precision f32`, else float64."""
        import torch
        return torch.float32 if (self.engine_mode == 'fast' or self.engine_precision == 'f32') else torch.float64

    def _upload(self, a, dev, pad=False):
        """The host array `a` as a table on `dev` in the engine's dtype.  With `pad`, under `-mode fast` a 2-D table
        gets zero columns up to a multiple of 4: the fast kernels move rows as 16-byte slices, the zero columns stay
        zero under their updates, and _host drops them."""
        import torch
        t = torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=self._engine_dtype())
        d = t.shape[-1]
        if not (pad and self.engine_mode == 'fast' and d % 4):
            return t
        padded = torch.zeros(t.shape[0], d + (4 - d % 4), device=dev, dtype=t.dtype)
        padded[:, :d] = t
        return padded

    def _tables_on_device(self):
        """The score_tables pair as contiguous float32 CUDA tensors on `engine=-device N`: what device_tables returns
        in the models that rank on the device."""
        import torch
        dev = torch.device('cuda', self.engine_device)
        return tuple(torch.from_numpy(np.ascontiguousarray(getattr(self, name), dtype=np.float32)).to(dev)
                     for name in self.score_tables)

    def _rating_csr_on_device(self, by, dev, with_vals):
        """The training ratings by 'user' or by 'item' (Rating.rating_csr) on `dev` for the ALS-family row solves:
        (rowptr, cols, vals in the engine's dtype, als_row_order), without vals unless `with_vals`."""
        import torch
        from .. import engine as E
        rowptr, cols, vals = self.data.rating_csr(by)
        csr = (torch.from_numpy(rowptr).to(dev), torch.from_numpy(cols).to(dev))
        if with_vals:
            csr += (torch.from_numpy(vals).to(device=dev, dtype=self._engine_dtype()),)
        return csr + (torch.from_numpy(E.als_row_order(rowptr)).to(dev),)

    def _host(self, t):
        """A device table as a float64 numpy array, without _upload's padding columns."""
        if t.dim() == 2:
            t = t[:, :self.emb_size]
        return np.ascontiguousarray(t.double().cpu().numpy())

    def printAlgorConfig(self):
        super(IterativeRecommender, self).printAlgorConfig()
        print('Embedding Dimension:', self.emb_size)
        print('Maximum Epoch:', self.maxEpoch)
        print('Regularization parameter: regU %.3f, regI %.3f, regB %.3f' % (self.regU, self.regI, self.regB))
        print('=' * 80)

    def initModel(self):
        # two draws from numpy's legacy global stream, P first (iterativeRecommender.py:37-38)
        self.P = np.random.rand(len(self.data.user), self.emb_size) / 3
        self.Q = np.random.rand(len(self.data.item), self.emb_size) / 3
        self.loss, self.lastLoss = 0, 0

    def updateLearningRate(self, epoch):
        if epoch > 1:
            self.lRate *= 1.05 if abs(self.lastLoss) > abs(self.loss) else 0.5
        if self.lRate > self.maxLRate > 0:
            self.lRate = self.maxLRate

    def predictForRating(self, u, i):
        known_u, known_i = self.data.containsUser(u), self.data.containsItem(i)
        if known_u and known_i:
            return self.P[self.data.user[u]].dot(self.Q[self.data.item[i]])
        if known_u:
            return self.data.userMeans[u]
        if known_i:
            return self.data.itemMeans[i]
        return self.data.globalMean

    def predictForRanking(self, u):
        if self.data.containsUser(u):
            U, V = (getattr(self, name) for name in self.score_tables)
            return V.dot(U[self.data.user[u]])
        return [self.data.globalMean] * self.num_items

    def shuffle_training_data(self):
        """`shuffle(self.data.trainingData)` (iterativeRecommender.py:101, deepRecommender.py:30)
        through the C MT19937 clone: the same swaps, the same generator state afterwards."""
        from ..engine import MT19937
        mt = MT19937()
        mt.setstate(random.getstate())
        perm = np.arange(len(self.data.trainingData), dtype=np.int32)
        mt.shuffle(perm)
        random.setstate(mt.getstate())
        data = self.data.trainingData
        self.data.trainingData[:] = [data[k] for k in perm.tolist()]
        return perm

    def isConverged(self, epoch):
        if isnan(self.loss):
            print('Loss = NaN or Infinity: current settings does not fit the recommender! Change the settings and try again!')
            sys.exit(-1)
        delta = self.lastLoss - self.loss
        if self.ranking.isMainOn():
            print('%s %s epoch %d: loss = %.4f, delta_loss = %.5f learning_Rate = %.5f'
                  % (self.modelName, self.foldInfo, epoch, self.loss, delta, self.lRate))
        else:
            m = self.rating_performance()
            print('%s %s epoch %d: loss = %.4f, delta_loss = %.5f learning_Rate = %.5f %5s %5s'
                  % (self.modelName, self.foldInfo, epoch, self.loss, delta, self.lRate, m[0].strip()[:11], m[1].strip()[:12]))
        converged = abs(delta) < 1e-3
        if not converged:
            self.updateLearningRate(epoch)
        self.lastLoss = self.loss
        self.shuffle_training_data()
        return converged

    def rating_performance(self):
        """iterativeRecommender.py:104-113.  While a model's tables are resident on the device it may set
        `_device_scores(tu, ti)`, the predictions of the test set's known (user id, item id) pairs computed there;
        every other line is predicted by predictForRating."""
        scored = {}
        if self._device_scores is not None:
            if not hasattr(self, '_test_pairs'):
                import torch
                dev = self._device()
                known = [k for k, (un, it, _) in enumerate(self.data.testData)
                         if self.data.containsUser(un) and self.data.containsItem(it)]
                tu = np.array([self.data.user[self.data.testData[k][0]] for k in known], dtype=np.int32)
                ti = np.array([self.data.item[self.data.testData[k][1]] for k in known], dtype=np.int32)
                self._test_pairs = (known, torch.from_numpy(tu).to(dev), torch.from_numpy(ti).to(dev))
            known, tu, ti = self._test_pairs
            scored = dict(zip(known, self._device_scores(tu, ti).double().cpu().tolist()))
        res = []
        for k, (user, item, rating) in enumerate(self.data.testData):
            pred = scored[k] if k in scored else self.predictForRating(user, item)
            res.append([user, item, rating, self.checkRatingBoundary(pred)])
        self.measure = Measure.ratingMeasure(res)
        return self.measure

    def ranking_performance(self, epoch):
        """In-training evaluation with best-epoch snapshot (iterativeRecommender.py:115-185)."""
        N = max(int(x) for x in self.ranking['-topN'].split(','))
        print('Evaluating...')
        recList = {}
        for user in self.data.testSet_u:
            scores = self.predictForRanking(user)
            for item in self.data.userRated(user)[0]:
                scores[self.data.item[item]] = 0
            ids, vals = find_k_largest(N, scores)
            recList[user] = list(zip([self.data.id2item[k] for k in ids], vals))
        measure = Measure.rankingMeasure(self.data.testSet_u, recList, [N])
        current = {}
        for m in measure[1:]:
            k, v = m.strip().split(':')
            current[k] = float(v)
        if self.bestPerformance:
            worse = sum(1 if self.bestPerformance[1][k] > current[k] else -1 for k in self.bestPerformance[1])
            if worse < 0:
                self.bestPerformance[1] = current
                self.bestPerformance[0] = epoch + 1
                self.saveModel()
        else:
            self.bestPerformance = [epoch + 1, current]
            self.saveModel()
        shown = [m.strip() for m in measure[1:]]
        best = self.bestPerformance[1]
        print('-' * 120)
        print('Quick Ranking Performance ' + self.foldInfo + ' (Top-' + str(N) + 'Item Recommendation)')
        print('*Current Performance*')
        print('Epoch:', str(epoch + 1) + ',', ' | '.join(shown))
        print('*Best Performance* ')
        print('Epoch:', str(self.bestPerformance[0]) + ',',
              'Precision:%s | Recall:%s | F1:%s | MDCG:%s' % (best['Precision'], best['Recall'], best['F1'], best['NDCG']))
        print('-' * 120)
        return shown
