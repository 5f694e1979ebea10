"""Shared pieces of the social rating models SoRec, RSTE, SocialMF, SoReg and SREE on the H100 engine.

Both train in the reference's order with the in-order kernels, in float64 (`engine=-precision f64`, the default) or
float32 (`-precision f32`; `-mode fast` runs the same kernels in float32, as WRMF and CoFactor do).  There is no
Hogwild path for them.  The host copies of the tables are refreshed after every epoch, since the reference's
evaluation and ranking read them."""
import numpy as np

from ...base.socialRecommender import SocialRecommender
from ._pointwise import PointwiseMF


def followee_csr(data, social):
    """The cleaned followee dicts as a CSR over the training users' ids, each row in the dict's insertion order:
    (rowptr int64 [U+1], cols int32, weights float64, denom float64 [U]).  denom[u] is the reference's
    `np.array(weights).sum()` (RSTE.py:51-52), summed by numpy in that order; 0 for a user who follows nobody."""
    U = len(data.user)
    rowptr = np.zeros(U + 1, np.int64)
    cols, weights, denom = [], [], np.zeros(U, np.float64)
    for k in range(U):
        name = data.id2user[k]
        ids, w = [], []
        for f, wf in social.getFollowees(name).items():
            if data.containsUser(f):
                ids.append(data.user[f])
                w.append(wf)
        cols.extend(ids)
        weights.extend(w)
        denom[k] = np.array(w).sum()
        rowptr[k + 1] = len(cols)
    return rowptr, np.array(cols, np.int32), np.array(weights, np.float64), denom


def follower_csr(data, social, values=None):
    """The cleaned follower dicts as a CSR over the training users' ids, each row in the dict's insertion order:
    (rowptr int64 [U+1], cols int32, vals float64).  vals are the relation weights, or values[u][g] (names) when
    `values` is given (SoReg's Sim)."""
    U = len(data.user)
    rowptr = np.zeros(U + 1, np.int64)
    cols, vals = [], []
    for k in range(U):
        name = data.id2user[k]
        for g, wg in social.getFollowers(name).items():
            if data.containsUser(g):
                cols.append(data.user[g])
                vals.append(wg if values is None else values[name][g])
        rowptr[k + 1] = len(cols)
    return rowptr, np.array(cols, np.int32), np.array(vals, np.float64)


def visit_order(data, social):
    """The user pass's visiting order: `social.user` (the first-appearance order of the relation list as read, before
    the cleaning) restricted to training users, as ids (SocialMF.py:26-27, SoReg.py:54-58)."""
    return np.array([data.user[name] for name in social.user if data.containsUser(name)], np.int32)


class SocialRatingMF(SocialRecommender):
    _upload = PointwiseMF._upload

    def _engine_dtype(self):
        import torch
        return torch.float32 if (self.engine_mode == 'fast' or self.engine_precision == 'f32') else torch.float64

    @staticmethod
    def _host(t):
        return np.ascontiguousarray(t.double().cpu().numpy())

    @staticmethod
    def _launch_width(n, depth):
        """n_warps of an in-order launch, from the stream's average parallel width (as PointwiseMF sizes K9)."""
        return int(min(2368, max(64, 16 * n / max(1, depth))))
