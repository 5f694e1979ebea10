"""CoFactor on the H100 engine -- drop-in for model/ranking/CoFactor.py of the reference (Liang et al. 2016: WRMF
plus a co-factorisation of the item-item SPPMI matrix).

`initModel` builds the SPPMI on the device (engine.sppmi_csr: co-occurrence counts with qrec_cooc_count, then
float64 PMI, shift, positive compaction and max-normalisation).  `trainModel` keeps X, Y, G, w, c on the device for
the whole run.  One epoch is
    Y^T Y (qrec_als_gram_*) -> every user row solved against Y, with the loss (qrec_als_solve_rows_*)
    -> X^T X -> the item sweep (qrec_cofactor_item_sweep_*),
then the reference's `epoch:` line.  The item sweep runs in item-id order and updates in place, exactly as the
reference's loop does, so the tables match the reference's float64 run to rounding; only the sums are grouped
differently.  Precision follows the `engine=` line: float64 tables by default, float32 tables with `-precision f32`
or `-mode fast` (the normal equations are float64 either way).

Reference behaviour kept as is:
  * the SPPMI: only items with at least `-filter` distinct users take part, a pair is kept when its number of common
    users is > filter (strict), the value is max(log((count*D) / (f_i*f_j)) - log(k), 0), kept when > 0, and all
    values are divided by their maximum; `-k` below 1 counts as 1.
  * X = 10*P, Y = 10*Q, then w = rand(I)/10, c = rand(I)/10, G = rand(I, d)/10 from numpy's global stream, in this
    order, at the start of trainModel.
  * alpha = 10 is hard-coded; Y is regularised with regU, G with `-gamma`; regI is unused.
  * G, w and c change only for items that have SPPMI contexts; w_i and c_i use Y_i and G_i from before item i's
    own solves.
  * the loss is WRMF's: sum (1 - x_u.y_i)^2 over the training entries with x_u before its solve, no regulariser.
  * there is no isConverged: exactly maxEpoch epochs run, with no reshuffle and no learning-rate change.
  * predictForRanking is Y.X[u].
"""
import numpy as np

from ...base.iterativeRecommender import IterativeRecommender
from ...util.config import OptionConf


class CoFactor(IterativeRecommender):
    ALPHA = 10.0
    score_tables = ('X', 'Y')

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(CoFactor, self).__init__(conf, trainingSet, testSet, fold)

    def readConfiguration(self):
        super(CoFactor, self).readConfiguration()
        extra = OptionConf(self.config['CoFactor'])
        self.negCount = int(extra['-k'])          # the number of negative samples
        if self.negCount < 1:
            self.negCount = 1
        self.regR = float(extra['-gamma'])
        self.filter = int(extra['-filter'])

    def printAlgorConfig(self):
        super(CoFactor, self).printAlgorConfig()
        print('Specified Arguments of', self.config['model.name'] + ':')
        print('k: %d' % self.negCount)
        print('regR: %.5f' % self.regR)
        print('filter: %d' % self.filter)
        print('=' * 80)

    def initModel(self):
        super(CoFactor, self).initModel()
        from ... import engine as E
        print('Constructing SPPMI matrix...')
        rowptr, cols, _ = self._rating_csr_on_device('item', self._device(), False)
        self.sppmi = E.sppmi_csr(rowptr, cols, self.num_users, self.negCount, self.filter)

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        self.X = self.P * 10
        self.Y = self.Q * 10
        self.w = np.random.rand(self.num_items) / 10
        self.c = np.random.rand(self.num_items) / 10
        self.G = np.random.rand(self.num_items, self.emb_size) / 10
        print('training...')
        X, Y, G, w, c = (self._upload(a, dev) for a in (self.X, self.Y, self.G, self.w, self.c))
        urp, ucol, uval, uord = self._rating_csr_on_device('user', dev, True)
        item_csr = self._rating_csr_on_device('item', dev, True)[:3]
        srp, scol, sval = self.sppmi
        sppmi = (srp, scol, sval.to(self._engine_dtype()))
        gram = torch.empty(self.emb_size, self.emb_size, dtype=torch.float64, device=dev)
        ws = E.als_gram_workspace(max(self.num_users, self.num_items), self.emb_size, dev)
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        stamps = torch.zeros(self.num_items, dtype=torch.int32, device=dev)
        epoch = 0
        while epoch < self.maxEpoch:
            loss.zero_()
            E.als_gram(Y, gram, ws)                                                   # YtY
            E.als_solve_rows(X, Y, gram, urp, ucol, uval, self.regU, self.ALPHA, uord, loss=loss)   # user loop
            E.als_gram(X, gram, ws)                                                   # XtX
            E.cofactor_item_sweep(Y, G, w, c, X, gram, item_csr, sppmi, self.regU, self.regR, self.ALPHA,
                                  stamps=stamps, sweep=epoch + 1)                     # item loop
            self.loss = float(loss.item())
            epoch += 1
            print('epoch:', epoch, 'loss:', self.loss)
        self.X, self.Y, self.G, self.w, self.c = (self._host(t) for t in (X, Y, G, w, c))

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
