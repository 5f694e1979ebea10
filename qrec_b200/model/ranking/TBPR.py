"""TBPR (social BPR with strong / weak ties) on the H100 engine -- drop-in for model/ranking/TBPR.py.

The reference's inner step `optimization(u, i, j)` (TBPR.py:44-52) is BPR.optimization statement for statement, so
the engine's K1 kernels run it unchanged; what is specific to TBPR is the HOST side, kept here with the
reference's semantics and random-number consumption:

  * tie strength = Jaccard index of the two users' followee sets, split at the median into strong and weak ties
    (TBPR.py:17-42);
  * per epoch the item sets a user's strong / weak ties have consumed and he has not, minus the items both kinds
    of tie have consumed, which form the "joint" set (TBPR.py:99-129);
  * per positive item i a preference chain  i > joint > weak > strong > unobserved  (only the levels that exist
    for the user), one `random.choice` per level in that order and a rejection loop for the unobserved item,
    giving consecutive (u, a, b) BPR steps (TBPR.py:131-160);
  * the epoch loss adds regU*|P|^2 + regI*|Q|^2 once PER USER, inside the user loop (TBPR.py:161) -- kept: in
    parity mode every user's chain is its own launch followed by the two table norms.
`optimization_theta` is never called by the reference's trainModel (theta_count stays 0), so theta only goes
through the clamping of TBPR.py:87-97; that code path is kept for the printed values.

engine=-mode parity (default): sequential semantics (qrec_bpr_sgd_ordered_*), float64 or float32.
engine=-mode fast: the whole epoch's chain steps in one user-major launch (qrec_bpr_sgd_usermajor_f32); the per-user
regulariser sum is then taken as (#users with positives) x the end-of-epoch norms (it only feeds the printed loss
and the learning-rate rule).
"""
import random
from collections import defaultdict

import numpy as np

from ...base.socialRecommender import SocialRecommender
from ...util import config


class TBPR(SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=list(), fold='[1]'):
        super(TBPR, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(TBPR, self).readConfiguration()
        self.regT = float(config.OptionConf(self.config['TBPR'])['-regT'])

    # ------------------------------------------------------------------ tie strength (TBPR.py:17-42)
    def initModel(self):
        super(TBPR, self).initModel()
        self.strength = defaultdict(dict)
        weights = []
        for u1 in self.social.user:
            mine = set(self.social.getFollowees(u1).keys())
            for u2 in self.social.getFollowees(u1):
                if u1 == u2:
                    continue
                theirs = set(self.social.getFollowees(u2).keys())
                s = len(mine.intersection(theirs)) / (len(mine.union(theirs)) + 0.0)
                self.strength[u1][u2] = s
                weights.append(s)
        weights.sort()
        self.weights = np.array(weights)
        self.theta = np.median(self.weights)
        self._split_ties()
        half = len(self.weights) // 2
        upper, lower = self.weights[half + 1:], self.weights[0:half]
        self.t_s = upper.sum() / (len(upper) + 0.0)
        self.t_w = lower.sum() / (len(lower) + 0.0)

    def _split_ties(self):
        self.strongTies, self.weakTies = defaultdict(dict), defaultdict(dict)
        for u1 in self.strength:
            for u2, s in self.strength[u1].items():
                (self.strongTies if s > self.theta else self.weakTies)[u1][u2] = s

    # ------------------------------------------------------------------ per-epoch host work
    def _clamp_theta(self):
        """TBPR.py:87-99."""
        if self.theta > self.weights.max():
            self.theta = self.weights.max() - 0.01
        if self.theta < self.weights.min():
            self.theta = self.weights.min() + 0.01
        try:
            above = [w for w in self.weights if w >= self.theta]
            below = [w for w in self.weights if w <= self.theta]
            self.t_s = sum(above) / len(above)
            self.t_w = sum(below) / len(below)
        except ZeroDivisionError:
            self.t_w = 0.01
            self.theta = 0.02
        self.g_theta = (self.t_s - self.theta) * (self.theta - self.t_w)

    def _consumed_by(self, ties, user):
        """Items (rating >= 1) of the users `user` is tied to that `user` has no positive feedback on, in
        first-seen order (the order the reference's dict gets them)."""
        out = {}
        mine = self.positiveSet[user]
        for friend in ties[user]:
            for item, r in self.data.trainSet_u[friend].items():
                if r >= 1 and item not in mine:
                    out[item] = 1
        return out

    def _item_sets(self):
        """jointSet / strongSet / weakSet of TBPR.py:103-129."""
        self.jointSet, self.strongSet, self.weakSet = defaultdict(dict), defaultdict(dict), defaultdict(dict)
        for u1 in self.social.user:
            if u1 in self.data.user:
                self.strongSet[u1] = self._consumed_by(self.strongTies, u1)
                self.weakSet[u1] = self._consumed_by(self.weakTies, u1)
        for u1 in self.social.user:
            if u1 in self.data.user:
                # same construction as the reference: the iteration order of this set decides which item a later
                # `choice` returns
                self.jointSet[u1] = dict.fromkeys(set(self.strongSet[u1].keys()).intersection(set(self.weakSet[u1].keys())), 1)
        for u1, joint in self.jointSet.items():
            if joint:
                self.strongSet[u1] = {k: 1 for k in self.strongSet[u1] if k not in joint}
                self.weakSet[u1] = {k: 1 for k in self.weakSet[u1] if k not in joint}

    def _sample_epoch(self):
        """The epoch's chain steps as int32 arrays (u, a, b) plus the number of steps of every user of positiveSet --
        TBPR.py:131-160 with the draws made by the native clone of CPython's generator (qrec_sample_tbpr_epoch): the
        interpreter's `random` state goes in and comes back, so the stream is the reference's draw for draw
        (`_sample_epoch_python` is the same loop in Python; tests/test_tbpr_cpu.py holds the two against each other and
        against the unmodified reference class)."""
        from ...engine import MT19937
        item_id, user_id = self.data.item, self.data.user
        csr = self.data.rated_csr()
        order = np.fromiter((user_id[x] for x in self.positiveSet), np.int32, len(self.positiveSet))
        # positiveSet[user] must be the positives RatedCSR lists (rating >= 1, insertion order)
        pools = []
        for level in (self.jointSet, self.weakSet, self.strongSet):
            rowptr = np.zeros(self.num_users + 1, np.int64)
            items = []
            for uid in range(self.num_users):
                keys = level.get(self.data.id2user[uid])
                if keys:
                    items.extend(item_id[k] for k in keys)
                rowptr[uid + 1] = len(items)
            pools.append((rowptr, np.asarray(items, dtype=np.int32)))
        mt = MT19937()
        mt.setstate(random.getstate())
        out = mt.sample_tbpr_epoch(csr, order, *pools)
        random.setstate(mt.getstate())
        return out

    def _sample_epoch_python(self):
        item_id, user_id = self.data.item, self.data.user
        item_list = list(item_id.keys())
        us, ia, ib, per_user = [], [], [], []
        for user, positives in self.positiveSet.items():
            u = user_id[user]
            levels = [list(self.jointSet[user].keys()), list(self.weakSet[user].keys()), list(self.strongSet[user].keys())]
            start = len(us)
            for item in positives:
                chain = [item_id[item]]
                for pool in levels:
                    if len(pool) > 0:
                        chain.append(item_id[random.choice(pool)])
                neg = random.choice(item_list)
                while neg in positives:
                    neg = random.choice(item_list)
                chain.append(item_id[neg])
                for a, b in zip(chain[:-1], chain[1:]):
                    us.append(u); ia.append(a); ib.append(b)
            per_user.append(len(us) - start)
        return (np.array(us, np.int32), np.array(ia, np.int32), np.array(ib, np.int32), np.array(per_user, np.int64))

    # ------------------------------------------------------------------ training
    def trainModel(self):
        import torch
        from ... import engine as E
        self.positiveSet = defaultdict(dict)
        for user in self.data.user:
            for item, r in self.data.trainSet_u[user].items():
                if r >= 1:
                    self.positiveSet[user][item] = 1
        dev = self._device()
        fast = self.engine_mode == 'fast'
        d = self.emb_size
        P, Q = self._upload(self.P, dev, pad=True), self._upload(self.Q, dev, pad=True)
        acc = torch.zeros(3, dtype=torch.float64, device=dev)
        print('Training...')
        epoch = 0
        while epoch < self.maxEpoch:
            self.theta_derivative, self.theta_count = 0, 0
            self._clamp_theta()
            print('Theta:', self.theta)
            print('g_theta:', self.g_theta)
            print('Preparing item sets...')
            self._item_sets()
            print('Computing...')
            u, a, b, per_user = self._sample_epoch()
            acc.zero_()
            if fast:
                rowptr = np.zeros(self.num_users + 1, np.int64)
                # users appear in positiveSet in id order (data.user is walked in id order): scatter their counts
                ids = np.fromiter((self.data.user[x] for x in self.positiveSet), np.int64, len(self.positiveSet))
                rowptr[ids + 1] = per_user
                rowptr = np.cumsum(rowptr)
                kernel = E.bpr_sgd_usermajor if P.shape[1] <= 128 else None
                da, db = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
                if kernel is not None and np.all(np.diff(u) >= 0):
                    kernel(P, Q, torch.from_numpy(rowptr).to(dev), da, db, self.lRate, self.regU, self.regI, acc[0:1])
                else:
                    E.bpr_sgd_batch(P, Q, torch.from_numpy(u).to(dev), da, db, self.lRate, self.regU, self.regI, acc[0:1])
                E.sumsq(P, acc[1:2]); E.sumsq(Q, acc[2:3])
                acc[1:3] *= float(len(per_user))
            else:
                lo = 0
                same = np.flatnonzero(a == b)                   # the unobserved item may repeat the chain's last member
                for n in per_user.tolist():                     # one user's chain steps, then the two norms (TBPR.py:161)
                    cuts = [lo] + [c for k in same[(same >= lo) & (same < lo + n)].tolist() for c in (k, k + 1)] + [lo + n]
                    for seg in range(0, len(cuts) - 1):
                        x, y = cuts[seg], cuts[seg + 1]
                        if y <= x:
                            continue
                        if seg % 2 == 1:                        # a single step with i == j
                            self._same_item_step(P, Q, int(u[x]), int(a[x]), acc)
                            continue
                        su, sa, sb = u[x:y], a[x:y], b[x:y]
                        wu, wi, wj = E.bpr_order_prepare(su, sa, sb, self.num_users, self.num_items)
                        E.bpr_sgd_ordered(P, Q, *(torch.from_numpy(t).to(dev) for t in (su, sa, sb, wu, wi, wj)),
                                          self.lRate, self.regU, self.regI, acc[0:1], n_warps=64)
                    E.sumsq(P, acc[1:2]); E.sumsq(Q, acc[2:3])
                    lo += n
            t = acc.cpu().numpy()
            self.loss = float(t[0] + self.regU * t[1] + self.regI * t[2])
            if self.theta_count > 0:                            # never true (see the module docstring); TBPR.py:162-171
                self.theta -= self.lRate * self.theta_derivative / self.theta_count
                self._split_ties()
            epoch += 1
            if not self.ranking.isMainOn():
                self.P = np.ascontiguousarray(P[:, :d].cpu().numpy())
                self.Q = np.ascontiguousarray(Q[:, :d].cpu().numpy())
            if self.isConverged(epoch):
                break
        self.P = np.ascontiguousarray(P[:, :d].cpu().numpy())
        self.Q = np.ascontiguousarray(Q[:, :d].cpu().numpy())

    def _same_item_step(self, P, Q, u, i, acc):
        """optimization(u, i, i) (TBPR.py:44-52 with j == i): numpy updates the shared row in place, statement by
        statement, so the row is raised, lowered by the same amount, and decayed twice; the score difference is
        exactly 0.  The K1 kernels take two DISTINCT item rows, so this (rare) step is applied here, on the device
        rows, in the reference's statement order."""
        import math
        g = self.lRate * (1 - 0.5)
        p, q = P[u], Q[i]
        q += g * p
        q -= g * p
        acc[0] += -math.log(0.5)
        p -= self.lRate * self.regU * p
        q -= self.lRate * self.regI * q
        q -= self.lRate * self.regI * q

    buildModel = trainModel
