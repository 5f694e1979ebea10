"""Shared pieces of the social rating models SoRec, RSTE, SocialMF, SoReg and SREE on the H100 engine.

Both train in the reference's order with the in-order kernels, in float64 (`engine=-precision f64`, the default) or
float32 (`-precision f32`; `-mode fast` runs the same kernels in float32, as WRMF and CoFactor do).  There is no
Hogwild path for them.  The host copies of the tables are refreshed after every epoch, since the reference's
evaluation and ranking read them."""
import numpy as np


def followee_csr(data, social, values=None):
    """The cleaned followee dicts as a CSR over the training users' ids, each row in the dict's insertion order:
    (rowptr int64 [U+1], cols int32, vals float64, denom float64 [U]).  vals are the relation weights, or values[u][f]
    (names) when `values` is given (SoReg's Sim).  denom[u] is the row's `np.array(vals).sum()`, which for the weights is
    the reference's (RSTE.py:51-52), summed by numpy in that order; 0 for a user who follows nobody."""
    U = len(data.user)
    rowptr = np.zeros(U + 1, np.int64)
    cols, vals, denom = [], [], np.zeros(U, np.float64)
    for k in range(U):
        name = data.id2user[k]
        ids, w = [], []
        for f, wf in social.getFollowees(name).items():
            if data.containsUser(f):
                ids.append(data.user[f])
                w.append(wf if values is None else values[name][f])
        cols.extend(ids)
        vals.extend(w)
        denom[k] = np.array(w).sum()
        rowptr[k + 1] = len(cols)
    return rowptr, np.array(cols, np.int32), np.array(vals, np.float64), denom


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


def user_pass_setup(model, P, values=None):
    """The K17 user pass of model's trust graph on the device table P: (args, g_val, n_warps).  args are the pass's
    arguments after P up to the follower values -- the visiting order, its schedule, the followee CSR with the relation
    weights or values[u][f] (`values`: SoReg's Sim), and the follower CSR -- and g_val the follower values when `values`
    is given, else None."""
    import torch
    from ... import engine as E
    rowptr, cols, f_val, _ = followee_csr(model.data, model.social, values)
    grp, gcols, g_val = follower_csr(model.data, model.social, values)
    visit = visit_order(model.data, model.social)
    pos, depth = E.social_order_prepare(visit, model.num_users, rowptr, cols, grp, gcols)
    t = lambda a: torch.from_numpy(a).to(P.device)                    # noqa: E731
    args = (t(visit), t(pos), t(rowptr), t(cols), model._upload(f_val, P.device), t(grp), t(gcols))
    return args, (None if values is None else model._upload(g_val, P.device)), E.ordered_warps(len(visit), depth)
