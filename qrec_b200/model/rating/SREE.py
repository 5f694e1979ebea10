"""SREE on the H100 engine -- drop-in for model/rating/SREE.py of the reference (Li et al. 2016): EE's rating pass
(K9 kind 5, see _euclidean.py) followed by the social pass over `social.user` restricted to training users
(SREE.py:48-61): each cleaned followee f of u in turn moves P[u] -= ((lr*alpha)*w_f)*(P[u]-P[f]) and adds
(alpha*w_f)*|P[u]-P[f]|^2 to the loss, from the row as the followees before it left it (K17, sree_user_pass)."""
from ...base.socialRecommender import SocialRecommender
from ...util import config
from ._euclidean import EuclideanMF
from ._social_rating import user_pass_setup


class SREE(EuclideanMF, SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=list(), fold='[1]'):
        super(SREE, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(SREE, self).readConfiguration()
        self.alpha = float(config.OptionConf(self.config['SREE'])['-alpha'])

    def _user_pass(self, P):
        from ... import engine as E
        args, _, n_warps = user_pass_setup(self, P)
        return lambda loss: E.sree_user_pass(P, *args, self.lRate, self.alpha, loss, n_warps=n_warps)
