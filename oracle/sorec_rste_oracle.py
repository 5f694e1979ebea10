"""CPU oracle for SoRec and RSTE (model/rating/SoRec.py, model/rating/RSTE.py) -- TEST INFRASTRUCTURE, NOT PRODUCT
CODE.  Only tests/ may import it.

Restates both models' epochs in plain numpy with the reference's own operations, so float64 runs are bit-identical
to it (tests/test_social_rating_cpu.py replays tests/golden/{sorec,rste}_filmtrust.npz, made by
oracle/gen_golden_sorec_rste.py from the unmodified reference).  With float32 tables it is the float32 yardstick of
the engine's kernels.  It also counts RSTE's wait numbers in pure Python, independently of qrec_rste_order_prepare.

`p = self.P[u]` is a numpy view in both models: the second row update reads the first row's new value.
"""
import math
from collections import defaultdict

import numpy as np


def clean_social(train_users, relation):
    """base/socialRecommender.py:7-41 over data/social.py:13-27: the followee / follower dicts (insertion order,
    the last weight of a repeated pair, its first position) and the relation list without the lines that name a
    user outside `train_users`."""
    followees, followers = defaultdict(dict), defaultdict(dict)
    for a, b, w in relation:
        followees[a][b] = w
        followers[b][a] = w
    for table in (followees, followers):
        for a in [a for a in table if a not in train_users]:
            del table[a]
        for a in table:
            for b in [b for b in table[a] if b not in train_users]:
                del table[a][b]
    kept = [r for r in relation if r[0] in train_users and r[1] in train_users]
    return followees, followers, kept


def sorec_edges(user_ids, followees, followers, relation):
    """SoRec.py:42-50: (u ids, v ids, targets weight*tuv) of the cleaned relation list, in its order."""
    us, vs, t = [], [], []
    for a, b, tuv in relation:
        vminus = len(followers[b]) if b in followers else 0
        uplus = len(followees[a]) if a in followees else 0
        try:
            weight = math.sqrt(vminus / (uplus + vminus + 0.0))
        except ZeroDivisionError:
            weight = 1
        us.append(user_ids[a])
        vs.append(user_ids[b])
        t.append(weight * tuv)
    return np.array(us, np.int32), np.array(vs, np.int32), t


def followee_lists(user_names, user_ids, followees):
    """Per user id: (followee ids, weights) as the reference's numpy arrays, in the dict's order (RSTE.py:45-52)."""
    out = []
    for name in user_names:
        ids, w = [], []
        for f, wf in (followees[name].items() if name in followees else ()):
            if f in user_ids:
                ids.append(user_ids[f])
                w.append(wf)
        out.append((np.array(ids), np.array(w)))
    return out


def initial_tables(seed, n_users, n_items, d, sorec):
    """P, Q (iterativeRecommender.py:37-38) and SoRec's Z (SoRec.py:17), drawn in that order from numpy's legacy
    global stream right after np.random.seed(seed)."""
    rs = np.random.RandomState(seed)
    P = rs.rand(n_users, d) / 3
    Q = rs.rand(n_items, d) / 3
    return (P, Q, rs.rand(n_users, d) / 10) if sorec else (P, Q)


def _cast(T, *xs):
    return [T(x) for x in xs]


def sorec_epoch(P, Q, Z, u, i, r, eu, ev, et, lr, reg_u, reg_i, reg_s, reg_z):
    """One SoRec epoch in place (SoRec.py:26-62); returns the loss as the reference leaves it before isConverged.
    dtype follows P (float64 = the reference)."""
    T = P.dtype.type
    lr, reg_u, reg_i, reg_s, reg_z = _cast(T, lr, reg_u, reg_i, reg_s, reg_z)
    loss = 0
    for k in range(len(u)):
        uu, ii = int(u[k]), int(i[k])
        error = T(r[k]) - P[uu].dot(Q[ii])
        loss += error ** 2
        p, q = P[uu], Q[ii]
        P[uu] += lr * (error * q - reg_u * p)
        Q[ii] += lr * (error * p - reg_i * q)
    for k in range(len(eu)):
        uu, vv = int(eu[k]), int(ev[k])
        euv = T(et[k]) - P[uu].dot(Z[vv])
        loss += reg_s * (euv ** 2)
        p, z = P[uu], Z[vv]
        P[uu] += lr * (reg_s * euv * z)
        Z[vv] += lr * (reg_s * euv * p - reg_z * z)
    loss += reg_u * (P * P).sum() + reg_i * (Q * Q).sum() + reg_z * (Z * Z).sum()
    return float(loss)


def rste_predict(P, Q, uu, ii, fl, alpha):
    """RSTE.py:41-62 for a known pair (ids)."""
    T = P.dtype.type
    alpha = T(alpha)
    idx, w = fl[uu]
    w = w.astype(P.dtype) if len(w) else w
    denom = w.sum()
    if denom != 0:
        f_pred = 0
        f_pred += w.dot(P[idx].dot(Q[ii]))
        return alpha * P[uu].dot(Q[ii]) + (T(1) - alpha) * f_pred / denom
    return P[uu].dot(Q[ii])


def rste_epoch(P, Q, u, i, r, fl, lr, reg_u, reg_i, alpha):
    """One RSTE epoch in place (RSTE.py:20-39); returns the loss as the reference leaves it before isConverged."""
    T = P.dtype.type
    lr, reg_u, reg_i, a = _cast(T, lr, reg_u, reg_i, alpha)
    loss = 0
    for k in range(len(u)):
        uu, ii = int(u[k]), int(i[k])
        error = T(r[k]) - rste_predict(P, Q, uu, ii, fl, alpha)
        loss += error ** 2
        p, q = P[uu], Q[ii]
        P[uu] += lr * (a * error * q - reg_u * p)
        Q[ii] += lr * (a * error * p - reg_i * q)
    loss += reg_u * (P * P).sum() + reg_i * (Q * Q).sum()
    return float(loss)


def rste_ranking(P, Q, uu, fl, alpha):
    """RSTE.py:66-83 for a known user id: the blend over all items, followee terms added one by one."""
    f_pred, denom = 0, 0
    idx, w = fl[uu]
    for f, wf in zip(idx.tolist(), w.tolist()):
        f_pred += wf * Q.dot(P[f])
        denom += wf
    if denom != 0:
        return alpha * Q.dot(P[uu]) + (1 - alpha) * f_pred / denom
    return Q.dot(P[uu])


def rste_waits(u, i, followees):
    """Pure-Python wait numbers of an RSTE stream: followees[u] lists u's followee ids (a self-follow allowed).
    Returns (wait_u, wait_i, wait_reads_u, follow_waits, depth); follow_waits[k] lists, per followee f != u of
    entry k, the number of earlier entries of user f."""
    writes_u, writes_i, reads = defaultdict(int), defaultdict(int), defaultdict(int)
    lw, lr, lq = defaultdict(int), defaultdict(int), defaultdict(int)
    wu, wi, wr, fw = [], [], [], []
    depth = 0
    for a, b in zip(list(u), list(i)):
        a, b = int(a), int(b)
        wu.append(writes_u[a])
        wi.append(writes_i[b])
        wr.append(reads[a])
        others = [f for f in followees[a] if f != a]
        fw.append([writes_u[f] for f in others])
        level = 1 + max([lw[a], lr[a], lq[b]] + [lw[f] for f in others])
        writes_u[a] += 1
        writes_i[b] += 1
        for f in others:
            reads[f] += 1
            lr[f] = max(lr[f], level)
        lw[a] = lq[b] = level
        depth = max(depth, level)
    return wu, wi, wr, fw, depth


def update_learning_rate(lr, max_lr, epoch, last_loss, loss):
    """iterativeRecommender.py:56-63."""
    if epoch > 1:
        if abs(last_loss) > abs(loss):
            lr *= 1.05
        else:
            lr *= 0.5
    if lr > max_lr > 0:
        lr = max_lr
    return lr
