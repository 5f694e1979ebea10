"""numpy restatement of one WRMF epoch (model/ranking/WRMF.py:19-67 of the reference), on CSR inputs.

Rows are solved with np.linalg.solve instead of the reference's inv(A).dot(b); the loss is summed in the same
user / entry order.  Test infrastructure only: the product never imports this module.
"""
import numpy as np

ALPHA = 10.0          # WRMF.py:34,55: hard-coded, the conf's -alpha is never read


def solve_side(X, Z, rowptr, cols, vals, lam, alpha=ALPHA, rows=None, with_loss=False):
    """Overwrites X[r] for every r in `rows` (default: all) with (Z^T Z + lam*I + alpha*sum v z z^T)^-1
    sum (1 + alpha*v) z over row r's entries; returns sum (1 - x_old.z)^2 when with_loss."""
    Z64 = np.asarray(Z, dtype=np.float64)
    G = Z64.T.dot(Z64)
    d = Z.shape[1]
    eye = lam * np.eye(d)
    loss = 0.0
    for r in (range(X.shape[0]) if rows is None else rows):
        c = cols[rowptr[r]:rowptr[r + 1]]
        v = np.asarray(vals[rowptr[r]:rowptr[r + 1]], dtype=np.float64)
        zr = Z64[c]
        if with_loss:
            x_old = np.asarray(X[r], dtype=np.float64)
            for k in range(len(c)):
                loss += (1.0 - x_old.dot(zr[k])) ** 2
        A = G + zr.T.dot(alpha * v[:, None] * zr) + eye
        b = ((1.0 + alpha * v)[:, None] * zr).sum(0) if len(c) else np.zeros(d)
        X[r] = np.linalg.solve(A, b)
    return loss


def epoch(X, Y, user_csr, item_csr, reg, alpha=ALPHA):
    """One epoch in place: users against Y (with the loss), then items against the new X.  Returns the loss."""
    loss = solve_side(X, Y, *user_csr, reg, alpha, with_loss=True)
    solve_side(Y, X, *item_csr, reg, alpha)
    return loss


def initial_tables(g):
    """X0, Y0 of a golden run: 10 * the P / Q draws of initModel (base/iterativeRecommender.py:37-38, P first) from
    the legacy numpy stream seeded with the run's seed (oracle/gen_golden_wrmf.py checks they are the recorded ones)."""
    r = np.random.RandomState(int(g['seed']))
    d = g['X_last'].shape[1]
    P = r.rand(len(g['user_names']), d) / 3
    Q = r.rand(len(g['item_names']), d) / 3
    return P * 10, Q * 10


def csr_from_dicts(rows_by_id, col_ids):
    """(rowptr, cols, vals) of a list of {column name: value} dicts (row id order), insertion order kept."""
    rowptr = np.zeros(len(rows_by_id) + 1, dtype=np.int64)
    cols, vals = [], []
    for k, row in enumerate(rows_by_id):
        for name, v in row.items():
            cols.append(col_ids[name])
            vals.append(float(v))
        rowptr[k + 1] = len(cols)
    return rowptr, np.array(cols, dtype=np.int32), np.array(vals, dtype=np.float64)


def golden_csrs(g):
    """User- and item-major CSRs of a golden run's training list, built the way the reference's
    trainSet_u / trainSet_i dicts are (data/rating.py): later duplicates overwrite the value in place."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    by_u = [dict() for _ in users]
    by_i = [dict() for _ in items]
    for un, it, r in zip(g['train_users'].tolist(), g['train_items'].tolist(), g['train_rating'].tolist()):
        by_u[users[un]][it] = r
        by_i[items[it]][un] = r
    return csr_from_dicts(by_u, items), csr_from_dicts(by_i, users)
