"""SBPR (social BPR, Zhao et al. CIKM'14) on the H100 engine -- drop-in for model/ranking/SBPR.py.

What the reference class does, path by path:

  * initModel (SBPR.py:12-29): PositiveSet[user] = the user's items with rating >= 1; FPSet[user][item] = how many
    of the user's followees (who are training users) consumed an item the user has not ("social feedback").  Kept
    statement for statement, including the defaultdict side effects the sampler's `len(self.FPSet[user])` relies on.
  * trainModel_tf (SBPR.py:103-134), the path its shipped configuration selects (`-tf`, config/SBPR.conf): minibatches
    of (u, i, k, j, S_uk) from `next_batch` (SBPR.py:69-101: positives in training-data order, one `choice` for the
    social item k, a rejection loop for the negative j -- Python's global `random`, consumed in exactly that order) and

        loss = - sum [ ln(sigmoid((x_ui - x_uk) / (S_uk + 1)) + 1e-6) + ln(sigmoid(x_uk - x_uj) + 1e-6) ]

    minimised by TF1 Adam over the two embedding tables.  The regulariser on the following source line
    (`+ self.regU * (...)`, SBPR.py:115) is a statement of its own and never reaches `loss`; it is absent here too.
    Here: K3 twice per minibatch -- qrec_bpr_grad_scatter_scaled_f32 on (u, i, k) with score scale 1 / (S_uk + 1),
    qrec_bpr_grad_scatter_f32 on (u, k, j) -- into the dense gradient buffers, then K4 (dense TF1 Adam: the
    IndexedSlices gradients of the three lookups are summed per row and TF1's sparse Adam still decays and applies every
    row's slots, which is the dense update with zeros elsewhere).
  * trainModel (SBPR.py:31-66), the numpy path: for the first user with social feedback it evaluates
    `self.FPSet[user][kItems]` with kItems a LIST (SBPR.py:47) and stops with `TypeError: unhashable type: 'list'`.
    The drop-in raises the same error at the same point of the life cycle; a data set in which no user has social
    feedback would run the reference's bias-augmented plain-BPR branch, which has no counterpart kernel (the item
    biases enter the sigmoid but are never trained) -- that corner raises QRecError instead of running on the host.
"""
from collections import defaultdict
from random import choice

import numpy as np

from ...base.socialRecommender import SocialRecommender


class SBPR(SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=None, fold='[1]'):
        super(SBPR, self).__init__(conf, trainingSet, testSet, relation, fold)

    def initModel(self):
        super(SBPR, self).initModel()
        print('Preparing item sets...')
        self.PositiveSet = defaultdict(dict)
        self.FPSet = defaultdict(dict)
        for user in self.data.user:
            mine = self.PositiveSet[user]
            for item, r in self.data.trainSet_u[user].items():
                if r >= 1:
                    mine[item] = 1
            if user in self.social.user:
                social = self.FPSet[user]
                for friend in self.social.getFollowees(user):
                    if friend in self.data.user:
                        for item in self.data.trainSet_u[friend]:
                            if item not in mine:
                                social[item] = social.get(item, 0) + 1

    # ------------------------------------------------------------------ numpy path (SBPR.py:31-66)
    def trainModel(self):
        from ...engine import QRecError
        self.b = np.random.random(self.num_items)          # the reference draws the biases before anything else
        print('Training...')
        for user in self.PositiveSet:
            if len(self.PositiveSet[user]) > 0 and len(self.FPSet[user]) > 0:
                # SBPR.py:47 `Suk = self.FPSet[user][kItems]` indexes a dict with the list of its own keys
                raise TypeError("unhashable type: 'list'")
        raise QRecError('SBPR.trainModel: no user has social feedback; the reference then runs a plain BPR step whose sigmoid '
                        'carries untrained item biases (SBPR.py:56-65) -- not built; use evaluation.setup -tf (config/SBPR.conf)')

    # ------------------------------------------------------------------ minibatch sampler (SBPR.py:69-101)
    def _social_csr(self):
        """FPSet as arrays over user ids: items in dict (insertion) order -- `choice(list(keys))` indexes that order --,
        their friend counts, and the same sets ascending for the membership test of the negative's rejection loop."""
        if getattr(self, '_fp_arrays', None) is None:
            item_id = self.data.item
            rowptr = np.zeros(self.num_users + 1, dtype=np.int64)
            items, counts, ordered = [], [], []
            for uid in range(self.num_users):
                social = self.FPSet[self.data.id2user[uid]]
                ids = [item_id[k] for k in social]
                items.extend(ids); counts.extend(social.values()); ordered.extend(sorted(ids))
                rowptr[uid + 1] = len(items)
            self._fp_arrays = (rowptr, np.asarray(items, dtype=np.int32), np.asarray(counts, dtype=np.int32),
                               np.asarray(ordered, dtype=np.int32))
        return self._fp_arrays

    def next_batch(self):
        """SBPR.py:69-101 with the per-row draws made by the native clone of CPython's generator
        (qrec_sample_sbpr_batch): Python's `random` state goes in before a batch and comes back after it, so the stream
        the interpreter sees is the reference's, draw for draw (`_next_batch_python` is the same loop in Python;
        tests/test_sbpr_cpu.py holds the two and the unmodified reference class against each other)."""
        import random
        from ...engine import MT19937
        csr = self.data.rated_csr()
        fp_rowptr, fp_items, fp_counts, fp_sorted = self._social_csr()
        u_all, i_all, _ = self.data.training_ids()
        for b in range(0, self.train_size, self.batch_size):
            u = np.ascontiguousarray(u_all[b:b + self.batch_size], dtype=np.int32)
            i = np.ascontiguousarray(i_all[b:b + self.batch_size], dtype=np.int32)
            mt = MT19937()
            mt.setstate(random.getstate())
            k, j, w = mt.sample_sbpr_batch(csr, fp_rowptr, fp_items, fp_counts, fp_sorted, u)
            random.setstate(mt.getstate())
            yield u, i, k, j, w

    def _next_batch_python(self):
        data, item_id, user_id = self.data.trainingData, self.data.item, self.data.user
        item_list = list(item_id.keys())
        batch_id = 0
        while batch_id < self.train_size:
            stop = min(batch_id + self.batch_size, self.train_size)
            u_idx, i_idx, f_idx, j_idx, weights = [], [], [], [], []
            for idx in range(batch_id, stop):
                user, item = data[idx][0], data[idx][1]
                i_idx.append(item_id[item])
                u_idx.append(user_id[user])
                social = self.FPSet[user]
                if len(social) == 0:
                    f_item = choice(item_list)
                    weights.append(0)
                else:
                    f_item = choice(list(social.keys()))
                    weights.append(social[f_item])
                f_idx.append(item_id[f_item])
                rated = self.data.trainSet_u[user]
                neg_item = choice(item_list)
                while neg_item in rated or neg_item in social:
                    neg_item = choice(item_list)
                j_idx.append(item_id[neg_item])
            batch_id = stop
            yield u_idx, i_idx, f_idx, j_idx, weights

    # ------------------------------------------------------------------ minibatch Adam (SBPR.py:103-134)
    def trainModel_tf(self):
        import torch
        from ... import engine as E
        dev = self._device()
        if not hasattr(self, 'batch_size'):
            self.batch_size = int(self.config['batch_size'])
        self.train_size = len(self.data.trainingData)
        d = self.emb_size
        dp = (d + 3) // 4 * 4                   # rows a multiple of 4 wide (SBPR.conf ships d=50 -> 52); zero columns stay zero
        U = torch.zeros(self.num_users, dp, device=dev)
        V = torch.zeros(self.num_items, dp, device=dev)
        U[:, :d] = torch.nn.init.trunc_normal_(torch.empty(self.num_users, d, device=dev), std=0.005, a=-0.01, b=0.01)
        V[:, :d] = torch.nn.init.trunc_normal_(torch.empty(self.num_items, d, device=dev), std=0.005, a=-0.01, b=0.01)
        mU, vU, mV, vV = (torch.zeros_like(t) for t in (U, U, V, V))
        gU, gV = torch.zeros_like(U), torch.zeros_like(V)
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        ids = lambda x: torch.from_numpy(np.asarray(x, dtype=np.int32)).to(dev)      # noqa: E731
        t = 0
        for epoch in range(self.maxEpoch):
            for n, (u, i, k, j, w) in enumerate(self.next_batch()):
                t += 1
                du, di, dk, dj = ids(u), ids(i), ids(k), ids(j)                 # int32 arrays from the native sampler
                scale = torch.from_numpy(1.0 / (np.asarray(w, dtype=np.float32) + np.float32(1.0))).to(dev)
                gU.zero_(); gV.zero_(); loss.zero_()
                E.bpr_grad_scatter_scaled(U, V, du, di, dk, scale, 1e-6, 0.0, gU, gV, loss)      # y_ik / (S_uk + 1)
                E.bpr_grad_scatter(U, V, du, dk, dj, 1e-6, 0.0, gU, gV, loss)                    # y_kj
                E.adam_dense_tf1(U, mU, vU, gU, self.lRate, t)
                E.adam_dense_tf1(V, mV, vV, gV, self.lRate, t)
                if n % 50 == 0:
                    print('training:', epoch + 1, 'batch', n, 'loss:', float(loss.item()))
        self.P = np.ascontiguousarray(U[:, :d].cpu().numpy())
        self.Q = np.ascontiguousarray(V[:, :d].cpu().numpy())
