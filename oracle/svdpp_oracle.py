"""numpy restatement of the reference's SVD++ epoch (model/rating/SVDPlusPlus.py:26-88) -- TEST INFRASTRUCTURE,
NOT PRODUCT CODE.  Only tests/ and tools/ may import it.

Two readings of the same per-entry step:
  * svdpp_sgd_sequential -- the literal loop, in the reference's expression order, so float64 results are
    bit-identical to the reference (tests/golden/svdpp_filmtrust.npz, oracle/gen_golden_svdpp.py);
  * svdpp_usermajor      -- the per-user closed form of the fast kernel (csrc/svdpp_step.cuh): one user's entries
    applied in order at O(W*d) instead of O(W^2*d), users taken in a given row order.

Per entry (u, i, r), with N(u) the user's distinct rated items in insertion order and w = |N(u)|:
    pred = (sum_{j in N(u)} Y[j] / w) . Q[i] + (((P[u].Q[i] + mean) + Bi[i]) + Bu[u]);  e = r - pred
    Bu[u] += lr*(e - regB*Bu[u]);  Bi[i] += lr*(e - regB*Bi[i])
    if w > 1:  Y[j] += lr*(e*q/(w-1) - regY*Y[j])  for j in N(u), j != i  (q = the old Q[i]);
               Q[i] += lr*e*sum_{j != i} Y_old[j] / (w-1)
    P[u] += lr*(e*Q[i] - regU*P[u]);  Q[i] += lr*(e*P[u] - regI*Q[i])     (Q[i] after the step above, new P[u])
"""
import numpy as np


def svdpp_sgd_sequential(P, Q, Y, Bu, Bi, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y, global_mean):
    """One pass over the entries (u[k], i[k], r[k]) in order, IN PLACE; returns sum(error^2) in float64.
    N(u) = cols[rowptr[u]:rowptr[u+1]] (the user's items in insertion order).  dtype follows P."""
    T = P.dtype.type
    lr, reg_u, reg_i, reg_b, reg_y, gm = (T(x) for x in (lr, reg_u, reg_i, reg_b, reg_y, global_mean))
    loss = 0.0
    for k in range(len(u)):
        uu, ii, rating = int(u[k]), int(i[k]), T(r[k])
        items = cols[rowptr[uu]:rowptr[uu + 1]]
        w = len(items)
        s = 0                                                       # SVDPlusPlus.py:76-80: sequential row sum
        for j in items:
            s = s + Y[j]
        pred = (s / T(w)).dot(Q[ii])
        pred = pred + (P[uu].dot(Q[ii]) + gm + Bi[ii] + Bu[uu])
        error = rating - pred
        loss += float(error) ** 2
        p, q = P[uu], Q[ii]                                         # views
        bu, bi = Bu[uu], Bi[ii]                                     # copies
        Bu[uu] += lr * (error - reg_b * bu)
        Bi[ii] += lr * (error - reg_b * bi)
        if w > 1:
            idx = [int(j) for j in items if j != ii]
            y = Y[idx]
            sm = y.sum(axis=0)
            Y[idx] += lr * (error * q / T(w - 1) - reg_y * y)
            Q[ii] += lr * error * sm / T(w - 1)
        P[uu] += lr * (error * q - reg_u * p)
        Q[ii] += lr * (error * p - reg_i * q)
    return loss


def epoch_loss(sq_err, P, Q, Y, Bu, Bi, reg_u, reg_i, reg_b, reg_y):
    """`self.loss` as the epoch ends (SVDPlusPlus.py:64-65)."""
    return float(sq_err + (reg_u * (P * P).sum() + reg_i * (Q * Q).sum() + reg_y * (Y * Y).sum()
                           + reg_b * ((Bu * Bu).sum() + (Bi * Bi).sum())))


def predict_rating(P, Q, Y, Bu, Bi, items, uu, ii, global_mean):
    """predictForRating (SVDPlusPlus.py:70-88) for a known pair; items: the user's item ids in insertion order."""
    s = 0
    for j in items:
        s = s + Y[j]
    pred = (s / len(items)).dot(Q[ii]) if len(items) else 0
    return pred + (P[uu].dot(Q[ii]) + global_mean + Bi[ii] + Bu[uu])


def user_entries(rowptr, cols, vals, row_order):
    """(u, i, r) of the CSR's entries, user by user in `row_order`, each user's items in CSR order."""
    rows = [int(x) for x in row_order]
    u = np.concatenate([np.full(rowptr[x + 1] - rowptr[x], x, np.int32) for x in rows]) if rows else np.empty(0, np.int32)
    sel = np.concatenate([np.arange(rowptr[x], rowptr[x + 1]) for x in rows]) if rows else np.empty(0, np.int64)
    return u, cols[sel].astype(np.int32), vals[sel]


def _user_closed_form(P, Q, Y, Bu, Bi, uu, items, rats, lr, reg_u, reg_i, reg_b, reg_y, gm):
    """One user's entries in order against the tables as they are now.  Returns (dQ rows, dBi, dY rows, new P row,
    new Bu, sum e^2); the caller applies the deltas (at once, or summed over the users in flight)."""
    W = len(items)
    c = 1.0 - lr * reg_y
    p = P[uu].astype(np.float64)
    bu = float(Bu[uu])
    Y0 = Y[items].astype(np.float64)
    S = Y0.sum(axis=0)
    B = np.zeros(Y.shape[1])
    dQ = np.zeros((W, Q.shape[1]))
    dBi = np.zeros(W)
    dY = np.zeros((W, Y.shape[1]))
    cW1 = c ** (W - 1)
    loss = 0.0
    for t in range(W):
        ii = items[t]
        q = Q[ii].astype(np.float64)
        bi = float(Bi[ii])
        yt = c ** t * Y0[t] + B
        e = float(rats[t]) - ((S / W).dot(q) + (p.dot(q) + gm + bi + bu))
        loss += e * e
        bu = bu + lr * (e - reg_b * bu)
        dBi[t] = lr * (e - reg_b * bi)
        qn = q
        if W > 1:
            v = lr * e * q / (W - 1)
            qn = q + lr * e * (S - yt) / (W - 1)
            dY[t] = (cW1 - 1.0) * Y0[t] + c ** (W - 1 - t) * ((1.0 - c) * B - v)
            S = c * (S - yt) + (W - 1) * v + yt
            B = c * B + v
        p = p + lr * (e * qn - reg_u * p)
        dQ[t] = qn + lr * (e * p - reg_i * qn) - q
    if W > 1:
        dY += B
    return dQ, dBi, dY, p, bu, loss


def svdpp_usermajor(P, Q, Y, Bu, Bi, rowptr, cols, vals, row_order, lr, reg_u, reg_i, reg_b, reg_y, global_mean,
                    users_in_flight=1):
    """The user-major epoch in closed form, IN PLACE (float64 arithmetic); returns sum(error^2).

    Users are taken from `row_order`; user u's entries are its CSR row (distinct items, one value each) in order.
    users_in_flight = 1: every user sees the tables left by the users before it -- equal to svdpp_sgd_sequential over
    user_entries(...) up to rounding.  users_in_flight = k > 1: consecutive groups of k users all read the tables as
    they stood before the group and their Q / Bi / Y deltas are summed (P and Bu rows are private to their user)."""
    k = max(1, int(users_in_flight))
    loss = 0.0
    order = [int(x) for x in row_order]
    for g0 in range(0, len(order), k):
        updates = []
        for uu in order[g0:g0 + k]:
            items = cols[rowptr[uu]:rowptr[uu + 1]].astype(np.int64)
            if len(items) == 0:
                continue
            out = _user_closed_form(P, Q, Y, Bu, Bi, uu, items, vals[rowptr[uu]:rowptr[uu + 1]], lr, reg_u, reg_i,
                                    reg_b, reg_y, global_mean)
            updates.append((uu, items, out))
        for uu, items, (dQ, dBi, dY, p, bu, l) in updates:
            np.add.at(Q, items, dQ.astype(Q.dtype))
            np.add.at(Bi, items, dBi.astype(Bi.dtype))
            np.add.at(Y, items, dY.astype(Y.dtype))
            P[uu] = p
            Bu[uu] = bu
            loss += l
    return loss


def initial_tables(g):
    """P0, Q0, Bu0, Bi0, Y0 of a golden run: the draws of SVDPlusPlus.initModel (SVDPlusPlus.py:20-24 after
    base/iterativeRecommender.py:37-38) from the legacy numpy stream seeded with the run's seed."""
    r = np.random.RandomState(int(g['seed']))
    nu, ni, d = len(g['user_names']), len(g['item_names']), g['P_last'].shape[1]
    P = r.rand(nu, d) / 3
    Q = r.rand(ni, d) / 3
    Bu = r.rand(nu)
    Bi = r.rand(ni)
    Y = r.rand(ni, d)
    return P, Q, Y, Bu, Bi


def golden_ids(g):
    """Id-mapped training list of a golden run (initial order) and the user CSR of trainSet_u (insertion order;
    a repeated (user, item) line keeps its first position and takes the last value)."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    u = np.array([users[x] for x in g['train_users'].tolist()], np.int32)
    i = np.array([items[x] for x in g['train_items'].tolist()], np.int32)
    by_u = [dict() for _ in users]
    for uu, ii, r in zip(u.tolist(), i.tolist(), g['train_rating'].tolist()):
        by_u[uu][ii] = r
    rowptr = np.zeros(len(users) + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum([len(row) for row in by_u])
    cols = np.array([j for row in by_u for j in row], dtype=np.int32)
    vals = np.array([v for row in by_u for v in row.values()], dtype=np.float64)
    return u, i, (rowptr, cols, vals), users, items
