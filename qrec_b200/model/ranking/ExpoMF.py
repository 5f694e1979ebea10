"""ExpoMF on the H100 engine -- drop-in for model/ranking/ExpoMF.py of the reference (Liang et al. 2016, "Modeling
User Exposure in Recommendation").

`trainModel` keeps theta, beta and mu on the device for the whole run.  One epoch is two launches of
qrec_expomf_solve_rows_f32 (engine.expomf_half_epoch):
    every user row against beta  ->  every item row against the new theta, fused with the exposure prior,
then mu is swapped with the prior's buffer.  Each CTA solves one row completely: it streams the whole other table,
weights every row by the exposure posterior of that (user, item) pair, lifts the observed entries to 1 and solves
the float64 system with a Cholesky factorization.  Nothing depends on the grid, so every run gives the same bits.

Reference behaviour kept as is:
  * initModel draws the base P and Q, then theta = 0.01*randn(U, d) and beta = 0.01*randn(I, d), in this order from
    numpy's global stream, each cast to float32; mu = 0.01 for every item.
  * lambda_y = 1, lambda_theta = lambda_beta = 1e-5, a = 1, b = 99 and EPS = 1e-8 are hard-coded; `reg.lambda` and
    `learnRate` are read and printed but never used.
  * the user half computes the posterior with the old theta, the current beta and mu by item; the item half with the
    old beta, the new theta and mu by item -- except when there are as many users as items: the reference picks the
    indexing with `mu.size == X.shape[0]`, so the item half then indexes mu by USER id.  This is reproduced.
  * the prior uses the new theta, the new beta and the old mu by item (always by item):
    mu_i = (a + sum_u A_ui - 1) / (a + b + U - 2), with A = 1 on the training entries.
  * theta, beta and mu are float32 in every `engine=` mode, as in the reference (`-precision` does not change them);
    the posteriors and both sides of every system are float64, and the solution is stored as float32.
  * there is no loss and no isConverged: exactly maxEpoch epochs run, with no reshuffle.  Each epoch prints
    `epoch #e`, `\tUpdating exposure prior...` and the mu it started from.
  * predictForRanking is beta.theta[u].
"""
import numpy as np

from ...base.iterativeRecommender import IterativeRecommender


class ExpoMF(IterativeRecommender):
    score_tables = ('theta', 'beta')

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(ExpoMF, self).__init__(conf, trainingSet, testSet, fold)

    def initModel(self):
        super(ExpoMF, self).initModel()
        self.lam_theta = 1e-5
        self.lam_beta = 1e-5
        self.lam_y = 1.0
        self.init_mu = 0.01
        self.a = 1.0
        self.b = 99.0
        self.init_std = 0.01
        self.theta = self.init_std * np.random.randn(self.num_users, self.emb_size).astype(np.float32)
        self.beta = self.init_std * np.random.randn(self.num_items, self.emb_size).astype(np.float32)
        self.mu = self.init_mu * np.ones(self.num_items, dtype=np.float32)

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        print('training...')
        theta, beta, mu = (torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
                           for a in (self.theta, self.beta, self.mu))
        mu_next = torch.empty_like(mu)
        urp, ucol, uord = self._rating_csr_on_device('user', dev, False)
        irp, icol, iord = self._rating_csr_on_device('item', dev, False)
        item_mu_by_row = self.num_users != self.num_items       # ExpoMF.py, _solve_batch: mu.size == X.shape[0]
        for epoch in range(self.maxEpoch):
            print('epoch #%d' % epoch)
            E.expomf_half_epoch(theta, beta, urp, ucol, mu, False, self.lam_theta / self.lam_y, self.lam_y, uord)
            E.expomf_half_epoch(beta, theta, irp, icol, mu, item_mu_by_row, self.lam_beta / self.lam_y, self.lam_y,
                                iord, mu_out=mu_next, a=self.a, b=self.b)
            print('\tUpdating exposure prior...')
            print(mu.cpu().numpy())
            mu, mu_next = mu_next, mu
        self.theta, self.beta, self.mu = (t.cpu().numpy() for t in (theta, beta, mu))

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
