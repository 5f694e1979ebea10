"""SocialMF on the H100 engine -- drop-in for model/rating/SocialMF.py of the reference (Jamali & Ester 2010).

An epoch is the reference's two passes, each one in-order launch:
  * the rating pass is K9 kind 4 over the training list in its current order: PMF's step on copies of both rows, so
    the item step reads the user row as it was before (SocialMF.py:15-24);
  * the user pass is K17 kind 0 over `social.user` restricted to training users (SocialMF.py:26-43): each user's row
    moves towards the weighted mean of its followees' rows, rl = P[u] - sum_f w_f P[f] / sum_f w_f (0 when the
    weights sum to 0), P[u] -= (lr*regS)*rl.
The loss is sum e^2 + regS*sum |rl|^2 + regU|P|^2 + regI|Q|^2, and training stops when isConverged says so, as in
the reference.  `-tf` is the base class's behaviour.  P and Q are float64 numpy arrays between epochs."""
from ...base.socialRecommender import SocialRecommender
from ._pointwise import ordered_rating_pass
from ._social_rating import user_pass_setup


class SocialMF(SocialRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, relation=None, fold='[1]'):
        super(SocialMF, self).__init__(conf, trainingSet, testSet, relation, fold)

    def readConfiguration(self):
        super(SocialMF, self).readConfiguration()

    def trainModel(self):
        import torch
        from ... import engine as E
        dev = self._device()
        P, Q = self._upload(self.P, dev), self._upload(self.Q, dev)
        social, _, pass_warps = user_pass_setup(self, P)
        acc = torch.zeros(4, dtype=torch.float64, device=dev)
        epoch = 0
        while epoch < self.maxEpoch:
            acc.zero_()
            ordered_rating_pass(self, E.SOCIALMF_RATINGS, P, Q, acc[0:1])
            E.social_user_pass(E.SOCIAL_PASS_KINDS['SocialMF'], P, *social, None, self.lRate, self.regS, acc[1:2],
                               n_warps=pass_warps)
            E.sumsq(P, acc[2:3]); E.sumsq(Q, acc[3:4])
            a = acc.cpu().numpy()
            self.loss = float(a[0] + a[1] + (self.regU * a[2] + self.regI * a[3]))
            self.P, self.Q = self._host(P), self._host(Q)
            epoch += 1
            if self.isConverged(epoch):
                break

    buildModel = trainModel
