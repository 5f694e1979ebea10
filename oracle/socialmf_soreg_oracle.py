"""CPU oracle for SocialMF and SoReg (model/rating/SocialMF.py, model/rating/SoReg.py) -- TEST INFRASTRUCTURE, NOT
PRODUCT CODE.  Only tests/ may import it.

Restates both models' epochs and SoReg's similarity construction in plain numpy / Python with the reference's own
operations, so float64 runs are bit-identical to it (tests/test_socialmf_soreg_cpu.py replays
tests/golden/{socialmf,soreg}_filmtrust.npz and socialmf_soreg_cases.npz, made by oracle/gen_golden_socialmf_soreg.py
from the unmodified reference).  With float32 tables it is the float32 yardstick of the engine's kernels.  It also
computes the user pass's schedule (visit positions and chain depth) in pure Python, independently of
qrec_social_order_prepare.

SocialMF copies both rows before its rating step; SoReg's rating step is PMF's (numpy views: the item step reads
the new user row).  The user pass visits `social.user` -- the relation list's first-appearance order as read, before
the cleaning -- and skips users who are not training users.
"""
from collections import defaultdict

import numpy as np

from oracle import knn_oracle as KO
from oracle.sorec_rste_oracle import _cast


def visit_ids(social_user_names, user_ids):
    """The visiting order as user ids: social.user restricted to training users."""
    return [user_ids[n] for n in social_user_names if n in user_ids]


def neighbour_lists(user_names, user_ids, table, values=None):
    """Per user id, (ids, values) of the cleaned dict `table` (followees or followers) in its order; values[u][v] (by
    name) replaces the relation weight when given."""
    out = []
    for name in user_names:
        ids, vals = [], []
        for v, w in (table[name].items() if name in table else ()):
            if v in user_ids:
                ids.append(user_ids[v])
                vals.append(w if values is None else values[name][v])
        out.append((ids, vals))
    return out


def soreg_similarities(user_names, followees, rows):
    """SoReg.py:21-36: Sim[user][f] = Sim[f][user] = (pearson_sp(rows[user], rows[f]) + weight(user, f)) / 2.0 for each
    training user in id order and each cleaned followee not met yet.  Returns (Sim, the pairs (user, f) in order)."""
    sim, pairs = defaultdict(dict), []
    for user in user_names:
        for f in (followees[user] if user in followees else {}):
            if user in sim and f in sim[user]:
                continue
            s = (KO.similarity(rows[user], rows[f], 'pcc') + followees[user][f]) / 2.0
            sim[user][f] = s
            sim[f][user] = s
            pairs.append((user, f))
    return sim, pairs


def rating_pass(P, Q, u, i, r, lr, reg_u, reg_i, copies, loss=0):
    """The rating pass in place; returns loss + sum e^2, added one by one.  copies: SocialMF's step on copies of both
    rows (K9 kind 4), else PMF's on views (kind 1)."""
    T = P.dtype.type
    lr, reg_u, reg_i = _cast(T, lr, reg_u, reg_i)
    for k in range(len(u)):
        uu, ii = int(u[k]), int(i[k])
        error = T(r[k]) - P[uu].dot(Q[ii])
        loss += error ** 2
        p, q = (P[uu].copy(), Q[ii].copy()) if copies else (P[uu], Q[ii])
        P[uu] += lr * (error * q - reg_u * p)
        Q[ii] += lr * (error * p - reg_i * q)
    return loss


def socialmf_user_pass(P, visit, fl, lr, reg_s, loss=0):
    """SocialMF.py:26-43 in place; returns loss + its loss terms, added one by one.  fl[u] = (followee ids, weights)."""
    T = P.dtype.type
    lr, reg_s = _cast(T, lr, reg_s)
    for uu in visit:
        f_pred, denom = 0, 0
        rl = np.zeros(P.shape[1], P.dtype)
        for f, w in zip(*fl[uu]):
            w = T(w)
            f_pred += w * P[f]
            denom += w
        if denom != 0:
            rl = P[uu] - f_pred / denom
        loss += reg_s * rl.dot(rl)
        P[uu] -= lr * reg_s * rl
    return loss


def soreg_user_pass(P, visit, fl, gl, lr, alpha, loss=0):
    """SoReg.py:54-72 in place; returns loss + its loss terms, added one by one.  fl[u] / gl[u] = (followee / follower
    ids, Sim values)."""
    T = P.dtype.type
    lr, alpha = _cast(T, lr, alpha)
    for uu in visit:
        sim_sum, f1 = 0, 0
        for f, s in zip(*fl[uu]):
            s = T(s)
            f1 += s * (P[uu] - P[f])
            sim_sum += s * ((P[uu] - P[f]).dot(P[uu] - P[f]))
            loss += sim_sum
        f2 = 0
        for g, s in zip(*gl[uu]):
            f2 += T(s) * (P[uu] - P[g])
        P[uu] += lr * (-alpha * (f1 + f2))
    return loss


def socialmf_epoch(P, Q, u, i, r, visit, fl, lr, reg_u, reg_i, reg_s):
    """One SocialMF epoch in place; returns the loss as the reference leaves it before isConverged."""
    loss = rating_pass(P, Q, u, i, r, lr, reg_u, reg_i, True)
    loss = socialmf_user_pass(P, visit, fl, lr, reg_s, loss)
    T = P.dtype.type
    loss += T(reg_u) * (P * P).sum() + T(reg_i) * (Q * Q).sum()
    return float(loss)


def soreg_epoch(P, Q, u, i, r, visit, fl, gl, lr, reg_u, reg_i, alpha):
    """One SoReg epoch in place; returns the loss as the reference leaves it before isConverged."""
    loss = rating_pass(P, Q, u, i, r, lr, reg_u, reg_i, False)
    loss = soreg_user_pass(P, visit, fl, gl, lr, alpha, loss)
    T = P.dtype.type
    loss += T(reg_u) * (P * P).sum() + T(reg_i) * (Q * Q).sum()
    return float(loss)


def schedule(visit, num_users, followees, followers):
    """Pure-Python schedule of the user pass: (pos, depth).  followees[u] / followers[u]: id lists."""
    pos = [-1] * num_users
    for k, uu in enumerate(visit):
        pos[uu] = k
    level, depth = [0] * num_users, 0
    for k, uu in enumerate(visit):
        before = [level[v] for v in list(followees[uu]) + list(followers[uu]) if v != uu and 0 <= pos[v] < k]
        level[uu] = 1 + max(before + [0])
        depth = max(depth, level[uu])
    return pos, depth
