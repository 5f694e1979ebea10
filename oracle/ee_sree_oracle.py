"""CPU oracle for EE and SREE (model/rating/EE.py, model/rating/SREE.py) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
Only tests/ may import it.

Restates both models' epochs in plain numpy / Python with the reference's own operations, in the order the kernels
apply them (K9 kind 5, the SREE pass of K17), so float64 runs are bit-identical to the reference
(tests/test_ee_sree_cpu.py replays tests/golden/{ee,sree}_filmtrust.npz and ee_sree_cases.npz, made by
oracle/gen_golden_ee_sree.py from the unmodified reference).  With float32 tables it is the float32 yardstick of the
engine's kernels.

EE's rating pass: e = r - (((globalMean + Bi[i]) + Bu[u]) - |P[u]-Q[i]|^2); the user step uses e + regU, the item
step e + regI and the user row after its step; both bias steps use the biases from before the entry.  SREE's user pass
visits `social.user` (first-appearance order of the relation list as read), skips users who are not training users,
and moves P[u] after every followee in turn.
"""
import numpy as np

from oracle.sorec_rste_oracle import _cast


def initial_biases(seed, n_users, n_items, d):
    """Bu, Bi (EE.py:11-12): drawn right after P and Q from numpy's legacy global stream seeded with `seed`."""
    rs = np.random.RandomState(seed)
    rs.rand(n_users, d)
    rs.rand(n_items, d)
    return rs.rand(n_users) / 10, rs.rand(n_items) / 10


def rating_pass(P, Q, Bu, Bi, u, i, r, lr, reg_u, reg_i, reg_b, global_mean):
    """EE.py:18-34 in place (the entries only); returns sum (e^2 + regU*dist), added one term at a time."""
    T = P.dtype.type
    lr, reg_u, reg_i, reg_b, gm = _cast(T, lr, reg_u, reg_i, reg_b, global_mean)
    loss = 0
    for k in range(len(u)):
        uu, ii = int(u[k]), int(i[k])
        dist = (P[uu] - Q[ii]).dot(P[uu] - Q[ii])
        error = T(r[k]) - (gm + Bi[ii] + Bu[uu] - dist)
        loss += error ** 2
        loss += reg_u * dist
        bu, bi = Bu[uu], Bi[ii]
        P[uu] -= lr * (error + reg_u) * (P[uu] - Q[ii])
        Q[ii] += lr * (error + reg_i) * (P[uu] - Q[ii])
        Bu[uu] += lr * (error - reg_b * bu)
        Bi[ii] += lr * (error - reg_b * bi)
    return loss


def bias_penalty(Bu, Bi, reg_b):
    """EE.py:35: regB*|Bu|^2 + regB*|Bi|^2."""
    reg_b = Bu.dtype.type(reg_b)
    return reg_b * (Bu * Bu).sum() + reg_b * (Bi * Bi).sum()


def sree_user_pass(P, visit, fl, lr, alpha, loss=0):
    """SREE.py:48-61 in place; returns loss + its terms, added one by one.  fl[u] = (followee ids, weights)."""
    T = P.dtype.type
    lr, alpha = _cast(T, lr, alpha)
    for uu in visit:
        for v, w in zip(*fl[uu]):
            w = T(w)
            p, z = P[uu], P[v]                   # views: a self-follow moves nothing
            P[uu] -= lr * alpha * w * (p - z)
            loss += alpha * w * (p - z).dot(p - z)
    return loss


def ee_epoch(P, Q, Bu, Bi, u, i, r, lr, reg_u, reg_i, reg_b, global_mean):
    """One EE epoch in place; returns the loss as the reference leaves it before isConverged."""
    loss = rating_pass(P, Q, Bu, Bi, u, i, r, lr, reg_u, reg_i, reg_b, global_mean)
    loss += bias_penalty(Bu, Bi, reg_b)
    return float(loss)


def sree_epoch(P, Q, Bu, Bi, u, i, r, visit, fl, lr, reg_u, reg_i, reg_b, global_mean, alpha):
    """One SREE epoch in place; returns the loss as the reference leaves it before isConverged."""
    loss = rating_pass(P, Q, Bu, Bi, u, i, r, lr, reg_u, reg_i, reg_b, global_mean)
    loss += bias_penalty(Bu, Bi, reg_b)
    return float(sree_user_pass(P, visit, fl, lr, alpha, loss))


def predict(P, Q, Bu, Bi, uu, ii, global_mean):
    """predictForRating (EE.py:81-87) of a known pair (ids)."""
    return global_mean + Bi[ii] + Bu[uu] - (P[uu] - Q[ii]).dot(P[uu] - Q[ii])


def ranking(P, Q, Bu, Bi, uu, global_mean):
    """predictForRanking (EE.py:89-96) of a known user id: the distance is added, so the farthest items rank first."""
    return ((Q - P[uu]) * (Q - P[uu])).sum(axis=1) + Bi + Bu[uu] + global_mean
