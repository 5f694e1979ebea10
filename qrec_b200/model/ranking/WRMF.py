"""WRMF on the H100 engine -- drop-in for model/ranking/WRMF.py of the reference (Hu et al., implicit-feedback ALS).

`trainModel` keeps X and Y on the device for the whole run.  One epoch (WRMF.py:19-67) is
    G = Y^T Y (qrec_als_gram_*) -> every user row solved against Y, with the loss (qrec_als_solve_rows_*)
    -> G = X^T X -> every item row solved against the new X,
then the reference's `epoch:` line and isConverged (which reshuffles trainingData, so a seeded run keeps the
MT19937 stream in step with the reference).  Given the other table every row's solve is independent, so the tables
match the reference's float64 run to rounding; only the loss is summed in a different order.
Precision follows the `engine=` line: float64 tables by default, float32 tables with `-precision f32` or
`-mode fast` (A and b are float64 either way).

Reference behaviour kept as is:
  * alpha = 10 is hard-coded (WRMF.py:34,55); the conf's `WRMF=-alpha 10 -lamba 1` is printed, never read.
  * both sides are regularised with regU (WRMF.py:41,60); regI is unused.
  * the loss is sum (1 - x_u.y_i)^2 over the training entries with x_u before its solve, no regulariser
    (WRMF.py:37-38,63); the item side adds nothing to it.
  * X = 10*P, Y = 10*Q from the usual initModel draws (WRMF.py:12-15).
"""
import numpy as np

from ...base.iterativeRecommender import IterativeRecommender


class WRMF(IterativeRecommender):
    ALPHA = 10.0

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(WRMF, self).__init__(conf, trainingSet, testSet, fold)

    def initModel(self):
        super(WRMF, self).initModel()
        self.X = self.P * 10
        self.Y = self.Q * 10

    def trainModel(self):
        import torch
        from ... import engine as E
        print('training...')
        dev = self._device()
        f32 = self.engine_mode == 'fast' or self.engine_precision == 'f32'
        dtype = torch.float32 if f32 else torch.float64
        X = torch.from_numpy(np.ascontiguousarray(self.X)).to(device=dev, dtype=dtype)
        Y = torch.from_numpy(np.ascontiguousarray(self.Y)).to(device=dev, dtype=dtype)
        sides = []
        for by in ('user', 'item'):
            rowptr, cols, vals = self.data.rating_csr(by)
            sides.append((torch.from_numpy(rowptr).to(dev), torch.from_numpy(cols).to(dev),
                          torch.from_numpy(vals).to(device=dev, dtype=dtype),
                          torch.from_numpy(E.als_row_order(rowptr)).to(dev)))
        G = torch.empty(self.emb_size, self.emb_size, dtype=torch.float64, device=dev)
        n_big = max(self.num_users, self.num_items)
        ws = torch.empty(max(1, int(E.lib.qrec_als_gram_workspace_bytes(n_big, self.emb_size))), dtype=torch.uint8,
                         device=dev)
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        epoch = 0
        while epoch < self.maxEpoch:
            loss.zero_()
            (urp, ucol, uval, uord), (irp, icol, ival, iord) = sides
            E.als_gram(Y, G, ws)                                                      # WRMF.py:22
            E.als_solve_rows(X, Y, G, urp, ucol, uval, self.regU, self.ALPHA, uord, loss=loss)   # :23-42
            E.als_gram(X, G, ws)                                                      # :44
            E.als_solve_rows(Y, X, G, irp, icol, ival, self.regU, self.ALPHA, iord)  # :45-61
            self.loss = float(loss.item())
            epoch += 1
            print('epoch:', epoch, 'loss:', self.loss)
            # with item.ranking off, isConverged scores ratings from P / Q, which WRMF never trains (as in the reference)
            if self.isConverged(epoch):
                break
        self._sync_host_tables(X, Y)

    buildModel = trainModel

    def _sync_host_tables(self, X, Y):
        self.X = np.ascontiguousarray(X.double().cpu().numpy())
        self.Y = np.ascontiguousarray(Y.double().cpu().numpy())

    def device_tables(self):
        import torch
        dev = torch.device('cuda', self.engine_device)
        return (torch.from_numpy(np.ascontiguousarray(self.X, dtype=np.float32)).to(dev),
                torch.from_numpy(np.ascontiguousarray(self.Y, dtype=np.float32)).to(dev))

    def predictForRanking(self, u):
        """WRMF.py:69-75"""
        if self.data.containsUser(u):
            return self.Y.dot(self.X[self.data.getUserId(u)])
        return [self.data.globalMean] * self.num_items
