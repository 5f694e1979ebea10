"""numpy restatement of CoFactor (model/ranking/CoFactor.py of the reference): the SPPMI matrix of initModel from a
sparse product, and one epoch of trainModel in reference order, on CSR inputs.

The SPPMI keeps the reference's definitions: only items with at least `filter` distinct users take part, on both
sides of a pair; a pair (i, j), j != i, is kept when its count of common users is > filter; f_i is the sum of row
i's kept counts and D the sum of all f; the value is max(log((count*D) / (f_i*f_j)) - log(k), 0), kept when > 0,
and every value is divided by the maximum.  The item sweep runs in item-id order and updates Y, G, w, c in place,
so a context c < i is read after its own update and c > i before it.  Contexts are visited in ascending id order
(the reference walks its dict's insertion order) and systems are solved with np.linalg.solve instead of
inv(A).dot(b).  Test infrastructure only: the product never imports this module.
"""
import math

import numpy as np
import scipy.sparse as sp

from . import wrmf_oracle as W

ALPHA = W.ALPHA       # CoFactor.py: `10 * r_ui` on both sides, hard-coded


def sppmi(item_rowptr, item_users, n_users, k, filt):
    """SPPMI CSR (rowptr int64, ascending cols int32, vals float64) and the raw co-occurrence CSR (rowptr, cols,
    counts int64) of the item-major CSR (item_rowptr, item_users: every item's distinct users)."""
    item_rowptr = np.asarray(item_rowptr, dtype=np.int64)
    n_items = len(item_rowptr) - 1
    k = max(int(k), 1)
    deg = np.diff(item_rowptr)
    B = sp.csr_matrix((np.ones(len(item_users), dtype=np.int64), np.asarray(item_users), item_rowptr),
                      shape=(n_items, n_users))
    B = sp.diags((deg >= filt).astype(np.int64), dtype=np.int64) @ B                 # ineligible items drop out of both sides
    C = (B @ B.T).tocoo()
    keep = (C.row != C.col) & (C.data > filt)
    C = sp.csr_matrix((C.data[keep], (C.row[keep], C.col[keep])), shape=(n_items, n_items))
    C.sort_indices()
    rows = np.repeat(np.arange(n_items), np.diff(C.indptr))
    f = np.asarray(C.sum(axis=1)).ravel().astype(np.float64)
    D = float(f.sum())
    logk = math.log(k)
    val = np.array([max(math.log((float(n) * D) / (f[a] * f[b])) - logk, 0.0)
                    for n, a, b in zip(C.data.tolist(), rows.tolist(), C.indices.tolist())])
    pos = val > 0
    out_rowptr = np.zeros(n_items + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows[pos], minlength=n_items), out=out_rowptr[1:])
    vals = val[pos]
    if len(vals):
        vals = vals / vals.max()
    return ((out_rowptr, C.indices[pos].astype(np.int32), vals),
            (C.indptr.astype(np.int64), C.indices.astype(np.int32), C.data.astype(np.int64)))


def item_sweep(Y, G, w, c, X, item_csr, sppmi_csr, reg, gamma, alpha=ALPHA, items=None):
    """The item half-epoch in place, items in id order (default: all).  Returns the number of items visited."""
    irp, icol, ival = item_csr
    srp, scol, sval = sppmi_csr
    X64 = np.asarray(X, dtype=np.float64)
    XtX = X64.T.dot(X64)
    d = X.shape[1]
    eye = np.eye(d)
    items = range(Y.shape[0]) if items is None else items
    for i in items:
        u = icol[irp[i]:irp[i + 1]]
        v = np.asarray(ival[irp[i]:irp[i + 1]], dtype=np.float64)
        xu = X64[u]
        ctx = scol[srp[i]:srp[i + 1]]
        m = np.asarray(sval[srp[i]:srp[i + 1]], dtype=np.float64)
        gam = np.asarray(G[ctx], dtype=np.float64)
        bet = np.asarray(Y[ctx], dtype=np.float64)
        w_c, c_c = np.asarray(w[ctx], dtype=np.float64), np.asarray(c[ctx], dtype=np.float64)
        w_i, c_i = float(w[i]), float(c[i])
        y_old, g_old = np.array(Y[i], dtype=np.float64), np.array(G[i], dtype=np.float64)   # copies: rows change below
        A = XtX + xu.T.dot(alpha * v[:, None] * xu) + reg * eye + gam.T.dot(gam)
        b = ((1.0 + alpha * v)[:, None] * xu).sum(0) + (((m - w_i) - c_c)[:, None] * gam).sum(0)
        Y[i] = np.linalg.solve(A, b)
        if len(ctx):
            G[i] = np.linalg.solve(bet.T.dot(bet) + gamma * eye, (((m - w_c) - c_i)[:, None] * bet).sum(0))
            w[i] = ((m - gam.dot(y_old)) - c_c).sum() / len(ctx)
            c[i] = ((m - bet.dot(g_old)) - w_c).sum() / len(ctx)
    return len(items)


def epoch(X, Y, G, w, c, user_csr, item_csr, sppmi_csr, reg, gamma, alpha=ALPHA):
    """One epoch in place: the WRMF user side against Y (with the loss), then the item sweep.  Returns the loss."""
    loss = W.solve_side(X, Y, *user_csr, reg, alpha, with_loss=True)
    item_sweep(Y, G, w, c, X, item_csr, sppmi_csr, reg, gamma, alpha)
    return loss


def initial_state(g, d):
    """X0, Y0, w0, c0, G0 of a golden run: 10 * the P / Q draws of initModel, then trainModel's w, c, G draws
    (CoFactor.py: rand(I)/10, rand(I)/10, rand(I, d)/10), from the legacy numpy stream seeded with the run's seed."""
    r = np.random.RandomState(int(g['seed']))
    nu, ni = len(g['user_names']), len(g['item_names'])
    P = r.rand(nu, d) / 3
    Q = r.rand(ni, d) / 3
    w = r.rand(ni) / 10
    c = r.rand(ni) / 10
    G = r.rand(ni, d) / 10
    return P * 10, Q * 10, w, c, G


def golden_csrs(g):
    """User- and item-major rating CSRs of a golden run (wrmf_oracle.golden_csrs)."""
    return W.golden_csrs(g)


def gauss_seidel_depth(sppmi_rowptr, sppmi_cols):
    """Length of the longest chain of the in-order item sweep: item i waits for every context c < i."""
    n = len(sppmi_rowptr) - 1
    depth = np.zeros(n, dtype=np.int64)
    for i in range(n):
        ctx = sppmi_cols[sppmi_rowptr[i]:sppmi_rowptr[i + 1]]
        ctx = ctx[ctx < i]
        depth[i] = 1 + (int(depth[ctx].max()) if len(ctx) else 0)
    return int(depth.max()) if n else 0
