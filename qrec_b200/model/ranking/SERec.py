"""SERec on the H100 engine -- drop-in for model/ranking/SERec.py of the reference (Chaney et al. 2015 / Wang et al.
2018, "Collaborative Filtering with Social Exposure: A Modular Approach to Social Recommendation").

SERec is ExpoMF with an exposure prior per (user, item) pair that grows with the user's number of followees.  The
reference holds that prior as a dense U x I matrix; it has the closed form
    mu(u, i) = (a + A_i + (s-1)*deg_u*A_i - 1) / (a + b + (s-1)*deg_u*A_i + U - 2)
with A_i the item's summed exposure posteriors and deg_u the user's followee count.  `trainModel` keeps theta, beta,
two A buffers (float64 [I]) and deg (int32 [U]) on the device for the whole run: O(U + I) state where the reference
needs three U x I float64 arrays per epoch.  One epoch is two launches of qrec_serec_solve_rows_f32
(engine.serec_half_epoch):
    every user row against beta  ->  every item row against the new theta, fused with the summed posteriors,
then the A buffers are swapped.  Each CTA solves one row completely (ExpoMF's fused row solve), evaluating the prior of
every pair from deg and A as it goes.  Nothing depends on the grid, so every run gives the same bits.

Reference behaviour kept as is:
  * initModel draws the base P and Q, then theta = 0.5*randn(U, d) and beta = 0.5*randn(I, d), in this order from
    numpy's global stream, each cast to float32; the prior starts at mu = 0.01 (float32) for every pair.
  * lambda_y = 0.01, lambda_theta = lambda_beta = 1e-5, a = 1, b = 99, s = 2.2 and EPS = 1e-8 are hard-coded;
    `reg.lambda` (including `-s`, printed by the social base class) and `learnRate` are read but never used.
  * the degree of a user counts the followees left in the cleaned `social.followees` (the row sums of the reference's
    0/1 matrix T), whatever the trust weights.
  * the user half uses mu[u, i] with the old theta and the current beta; the item half uses mu[u, i] with the old beta
    and the new theta -- except when there are as many users as items: the reference picks the branch with
    `mu.shape[1] == X.shape[0]`, so the item half then reads mu[i, u] (deg of the item's id, A of the user's).  This
    is reproduced.
  * A is summed from the new theta, the new beta and the OLD mu[u, i] (always by user row), with A = 1 on the training
    entries; the next epoch's prior is formed from it in float64.  The kernel forms deg_u * A_i as one product where
    the reference's T.dot adds A_i deg_u times (a few ulps apart for deg_u >= 7).
  * theta and beta are float32 in every `engine=` mode, as in the reference (`-precision` does not change them); the
    posteriors and both sides of every system are float64, and the solution is stored as float32.
  * there is no loss and no isConverged: exactly maxEpoch epochs run, with no reshuffle.  Each epoch prints
    `epoch #e`, the U x I mu it started from (float32 in the first epoch, float64 after) and
    `\tUpdating exposure prior...`.  The matrix print is byte for byte numpy's without building the matrix: a
    summarised print shows only the edge rows and columns, which are computed on the host from deg and A, with the
    reference's repeated sum for deg_u * A_i.
  * predictForRanking is beta.theta[u].
"""
import numpy as np

from ...base.socialRecommender import SocialRecommender


def mu_entries(A, deg, n_users, a=1.0, b=99.0, s=2.2, init_mu=0.01, n_items=None):
    """The reference's mu for the users with degrees deg and the items with summed posteriors A, as it computes them:
    (a + A + (s-1)*S - 1) / (a + b + (s-1)*S + U - 2) with S = A added to itself deg times (T.dot of the tiled A).
    A None: the first epoch's init_mu * ones(float32), n_items columns."""
    deg = np.asarray(deg, dtype=np.int64)
    if A is None:
        return init_mu * np.ones((deg.shape[0], n_items), dtype=np.float32)
    A = np.asarray(A, dtype=np.float64)
    S = np.zeros((deg.shape[0], A.shape[0]))
    for k in range(int(deg.max()) if deg.size else 0):
        S[deg > k] += A
    return (a + A[None, :] + (s - 1) * S - 1) / (a + b + (s - 1) * S + n_users - 2)


def mu_text(A, deg, n_items, **kw):
    """str() of the reference's U x I mu without building it when numpy would summarise it: numpy formats a
    summarised array from its leading and trailing `edgeitems` rows and columns only, so those (with one filler row or
    column where an axis is cut) are printed with summarising forced on."""
    U = len(deg)
    opts = np.get_printoptions()
    if U * n_items <= opts['threshold']:
        return str(mu_entries(A, deg, U, n_items=n_items, **kw))
    e = opts['edgeitems']

    def edges(n):
        return np.arange(n) if n <= 2 * e else np.concatenate([np.arange(e + 1), np.arange(n - e, n)])
    rows, cols = edges(U), edges(n_items)
    block = mu_entries(None if A is None else np.asarray(A)[cols], np.asarray(deg)[rows], U, n_items=len(cols), **kw)
    with np.printoptions(threshold=0):
        return str(block)


class SERec(SocialRecommender):
    score_tables = ('theta', 'beta')

    def __init__(self, conf, trainingSet=None, testSet=None, relation=None, fold='[1]'):
        super(SERec, self).__init__(conf, trainingSet, testSet, relation, fold)

    def initModel(self):
        super(SERec, self).initModel()
        self.lam_theta = 1e-5
        self.lam_beta = 1e-5
        self.lam_y = 0.01
        self.init_mu = 0.01
        self.a = 1.0
        self.b = 99.0
        self.s = 2.2
        self.init_std = 0.5
        self.theta = self.init_std * np.random.randn(self.num_users, self.emb_size).astype(np.float32)
        self.beta = self.init_std * np.random.randn(self.num_items, self.emb_size).astype(np.float32)
        self.deg = np.zeros(self.num_users, dtype=np.int32)          # row sums of SERec.py's T
        for user in self.social.followees:
            self.deg[self.data.user[user]] = len(self.social.followees[user])
        self.A = None                                                 # summed posteriors; None: mu = init_mu

    def mu_rows(self, users):
        """Rows of the current U x I prior for the users listed (as the reference would hold them)."""
        return mu_entries(self.A, self.deg[np.asarray(users)], self.num_users, self.a, self.b, self.s, self.init_mu,
                          self.num_items)

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        print('training...')
        theta, beta = (torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
                       for a in (self.theta, self.beta))
        deg = torch.from_numpy(self.deg).to(dev)
        asum, asum_next = None, torch.empty(self.num_items, dtype=torch.float64, device=dev)
        urp, ucol, uord = self._rating_csr_on_device('user', dev, False)
        irp, icol, iord = self._rating_csr_on_device('item', dev, False)
        item_rows_are_users = self.num_users == self.num_items      # SERec.py, _solve_batch: mu.shape[1] == X.shape[0]
        kw = dict(mu0=self.init_mu, a=self.a, b=self.b, s=self.s)
        for epoch in range(self.maxEpoch):
            print('epoch #%d' % epoch)
            E.serec_half_epoch(theta, beta, urp, ucol, asum, deg, True, self.lam_theta / self.lam_y, self.lam_y, uord,
                               **kw)
            E.serec_half_epoch(beta, theta, irp, icol, asum, deg, item_rows_are_users, self.lam_beta / self.lam_y,
                               self.lam_y, iord, asum_out=asum_next, **kw)
            print(mu_text(self.A, self.deg, self.num_items, a=self.a, b=self.b, s=self.s, init_mu=self.init_mu))
            print('\tUpdating exposure prior...')
            self.A = asum_next.cpu().numpy()
            if asum is None:
                asum = torch.empty_like(asum_next)
            asum, asum_next = asum_next, asum
        self.theta, self.beta = (t.cpu().numpy() for t in (theta, beta))

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
