"""SoRec on the H100 engine -- drop-in for model/rating/SoRec.py of the reference (Ma et al. 2008).

An epoch is the reference's two passes, each one in-order launch:
  * the rating pass is PMF's step, K9 kind 1 over the training list in its current order (SoRec.py:30-40);
  * the trust-edge pass is K9 kind 3 over the cleaned relation list in order on the tables (P, Z)
    (SoRec.py:42-60).  The target of edge (u, v) is weight*tuv with weight = sqrt(|followers(v)| /
    (|followees(u)| + |followers(v)| + 0.0)) over the cleaned dicts, computed here in Python floats.
The loss is sum e^2 + regS*sum e_uv^2 + regU|P|^2 + regI|Q|^2 + regZ|Z|^2, and training stops when isConverged
says so, as in the reference.  P, Q and Z are float64 numpy arrays between epochs."""
import math

import numpy as np

from ...base.socialRecommender import SocialRecommender
from ...util import config
from ._pointwise import ordered_rating_pass


class SoRec(SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=list(), fold='[1]'):
        super(SoRec, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(SoRec, self).readConfiguration()
        self.regZ = float(config.OptionConf(self.config['SoRec'])['-z'])

    def initModel(self):
        super(SoRec, self).initModel()
        self.Z = np.random.rand(self.data.trainingSize()[0], self.emb_size) / 10   # right after P and Q

    def printAlgorConfig(self):
        super(SoRec, self).printAlgorConfig()
        print('Specified Arguments of', self.config['model.name'] + ':')
        print('regZ: %.3f' % self.regZ)
        print('=' * 80)

    def edge_targets(self):
        """The relation list as id arrays (u, v) and its targets weight*tuv (SoRec.py:45-50)."""
        us, vs, targets = [], [], []
        for u, v, tuv in self.social.relation:
            vminus = len(self.social.getFollowers(v))
            uplus = len(self.social.getFollowees(u))
            try:
                weight = math.sqrt(vminus / (uplus + vminus + 0.0))
            except ZeroDivisionError:
                weight = 1
            us.append(self.data.user[u])
            vs.append(self.data.user[v])
            targets.append(weight * tuv)
        return np.array(us, np.int32), np.array(vs, np.int32), np.array(targets, np.float64)

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        U = self.num_users
        P, Q, Z = (self._upload(t, dev) for t in (self.P, self.Q, self.Z))
        eu, ev, et = self.edge_targets()
        ewu, ewv = E.mf_order_prepare(eu, ev, U, U)
        edges = [torch.from_numpy(a).to(dev) for a in (eu, ev, ewu, ewv)]
        dt_edge = self._upload(et, dev)
        edge_warps = E.ordered_warps(len(eu), E.mf_order_depth(eu, ev, U, U))
        acc = torch.zeros(5, dtype=torch.float64, device=dev)
        epoch = 0
        while epoch < self.maxEpoch:
            acc.zero_()
            ordered_rating_pass(self, 1, P, Q, acc[0:1])
            E.mf_sgd_ordered(E.SOREC_EDGES, P, Z, edges[0], edges[1], dt_edge, edges[2], edges[3], self.lRate,
                             self.regS, self.regZ, acc[1:2], n_warps=edge_warps)
            E.sumsq(P, acc[2:3]); E.sumsq(Q, acc[3:4]); E.sumsq(Z, acc[4:5])
            a = acc.cpu().numpy()
            self.loss = float(a[0] + a[1] + (self.regU * a[2] + self.regI * a[3] + self.regZ * a[4]))
            self.P, self.Q, self.Z = self._host(P), self._host(Q), self._host(Z)
            epoch += 1
            if self.isConverged(epoch):
                break

    buildModel = trainModel
