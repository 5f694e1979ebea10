"""SREE on the H100 engine -- drop-in for model/rating/SREE.py of the reference (Li et al. 2016): EE's rating pass
(K9 kind 5, see _euclidean.py) followed by the social pass over `social.user` restricted to training users
(SREE.py:48-61): each cleaned followee f of u in turn moves P[u] -= ((lr*alpha)*w_f)*(P[u]-P[f]) and adds
(alpha*w_f)*|P[u]-P[f]|^2 to the loss, from the row as the followees before it left it (K17, sree_user_pass)."""
from ...util import config
from ._euclidean import EuclideanMF
from ._social_rating import SocialRatingMF, follower_csr, followee_csr, visit_order


class SREE(EuclideanMF, SocialRatingMF):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=list(), fold='[1]'):
        super(SREE, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(SREE, self).readConfiguration()
        self.alpha = float(config.OptionConf(self.config['SREE'])['-alpha'])

    def _user_pass(self, P, dev, dtype):
        import torch
        from ... import engine as E
        rowptr, cols, w, _ = followee_csr(self.data, self.social)
        grp, gcols, _ = follower_csr(self.data, self.social)
        visit = visit_order(self.data, self.social)
        pos, depth = E.social_order_prepare(visit, self.num_users, rowptr, cols, grp, gcols)
        t = lambda a: torch.from_numpy(a).to(dev)                    # noqa: E731
        args = (t(visit), t(pos), t(rowptr), t(cols), torch.from_numpy(w).to(device=dev, dtype=dtype), t(grp), t(gcols))
        n_warps = self._launch_width(len(visit), depth)
        return lambda loss: E.sree_user_pass(P, *args, self.lRate, self.alpha, loss, n_warps=n_warps)
