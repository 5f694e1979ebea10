"""float64 numpy restatement of ExpoMF (model/ranking/ExpoMF.py of the reference), on CSR inputs.

The reference computes the exposure posterior and each row's Gram X^T (A X) in float32 and solves in float64; here
every product, sum and solve is float64 and only the stored rows (theta, beta, mu: float32 tables, as in the
reference) are rounded, as the engine does.  One epoch: every user against beta (mu by item), every item against the
new theta (mu by item, or by USER when the two tables have as many rows -- the reference's `mu.size == X.shape[0]`
test in _solve_batch), then the exposure prior from the new tables and the old mu.  Test infrastructure only: the
product never imports this module.
"""
import math

import numpy as np

LAM = 1e-5            # ExpoMF.py: lam_theta = lam_beta = 1e-5, lam_y = 1, used as lam / lam_y
LAM_Y = 1.0
A_PRIOR, B_PRIOR = 1.0, 99.0
EPS = 1e-8
INIT_MU, INIT_STD = 0.01, 0.01


def exposure(S, mu, lam_y=LAM_Y):
    """Posterior of exposure (ExpoMF.py: a_row_batch) of the dot products S with priors mu, before the lift."""
    S = np.asarray(S, dtype=np.float64)
    mu = np.asarray(mu, dtype=np.float64)
    p = math.sqrt(lam_y / 2 / np.pi) * np.exp(-lam_y * S ** 2 / 2)
    return (p + EPS) / (p + EPS + (1 - mu) / mu)


def solve_row(x_old, Z, cols, mu_row, lam=LAM, lam_y=LAM_Y):
    """The new value of one row (float64), or None when its system is not positive definite.  x_old: the row before
    the update; Z: the other table; cols: the row's observed columns; mu_row: a scalar (mu by row) or one prior per
    row of Z (mu by column)."""
    Z64 = np.asarray(Z, dtype=np.float64)
    A = exposure(Z64.dot(np.asarray(x_old, dtype=np.float64)), mu_row, lam_y)
    A = np.broadcast_to(A, (Z64.shape[0],)).copy()
    A[np.asarray(cols, dtype=np.int64)] = 1.0
    B = (Z64.T * A).dot(Z64) + lam * np.eye(Z64.shape[1])
    try:
        np.linalg.cholesky(B)
    except np.linalg.LinAlgError:
        return None
    return np.linalg.solve(B, Z64[np.asarray(cols, dtype=np.int64)].sum(0))


def solve_side(X, Z, rowptr, cols, mu, mu_by_row, lam=LAM, lam_y=LAM_Y, rows=None):
    """ExpoMF.py: recompute_factors in place on X (rows rounded to X's dtype) against Z; every row reads its own old
    value only.  mu is indexed by X's row (mu_by_row) or by Z's row.  Returns the number of rows left unchanged
    because their system was not positive definite."""
    mu64 = np.asarray(mu, dtype=np.float64)
    failed = 0
    for r in (range(X.shape[0]) if rows is None else rows):
        x = solve_row(X[r], Z, cols[rowptr[r]:rowptr[r + 1]], mu64[r] if mu_by_row else mu64, lam, lam_y)
        if x is None:
            failed += 1
        else:
            X[r] = x
    return failed


def prior(theta, beta, mu, user_csr, a=A_PRIOR, b=B_PRIOR, lam_y=LAM_Y):
    """ExpoMF.py: _update_expo -- the new mu (float64) from the posteriors of theta.beta with the old mu by item,
    1 on the training entries."""
    rowptr, cols = user_csr[0], user_csr[1]
    n_users = theta.shape[0]
    A = exposure(np.asarray(theta, dtype=np.float64).dot(np.asarray(beta, dtype=np.float64).T), mu[None, :], lam_y)
    rows = np.repeat(np.arange(n_users), np.diff(rowptr))
    A[rows, np.asarray(cols, dtype=np.int64)] = 1.0
    return (a + A.sum(0) - 1) / (a + b + n_users - 2)


def prior_rows(X, Z, rowptr, cols, mu, a=A_PRIOR, b=B_PRIOR, lam_y=LAM_Y, rows=None):
    """The same prior from the rows' side, as the item half of the engine computes it: for each row r of X (an item)
    against every row of Z (the users), (a + sum_k A_k - 1) / (a + b + len(Z) - 2) with A from x_r.z_k and mu[r],
    1 on row r's observed columns.  Returns a float64 array with one entry per row listed (default: all)."""
    Z64 = np.asarray(Z, dtype=np.float64)
    out = []
    for r in (range(X.shape[0]) if rows is None else rows):
        A = exposure(Z64.dot(np.asarray(X[r], dtype=np.float64)), float(mu[r]), lam_y)
        A[np.asarray(cols[rowptr[r]:rowptr[r + 1]], dtype=np.int64)] = 1.0
        out.append((a + A.sum() - 1) / (a + b + Z64.shape[0] - 2))
    return np.array(out, dtype=np.float64)


def epoch(theta, beta, mu, user_csr, item_csr, mu_by_row=None, lam=LAM, lam_y=LAM_Y, a=A_PRIOR, b=B_PRIOR):
    """One epoch in place on theta, beta, mu (float32 arrays).  mu_by_row: how the item half indexes mu; None follows
    the reference (by item, unless users and items are as many -- then by user).  Returns the failed rows."""
    failed = solve_side(theta, beta, user_csr[0], user_csr[1], mu, False, lam, lam_y)
    if mu_by_row is None:
        mu_by_row = theta.shape[0] != beta.shape[0]
    failed += solve_side(beta, theta, item_csr[0], item_csr[1], mu, mu_by_row, lam, lam_y)
    mu[:] = prior(theta, beta, mu, user_csr, a, b, lam_y)
    return failed


def initial_state(g, d):
    """theta0, beta0, mu0 of a golden run (float32): the base initModel's P / Q draws, then 0.01 * randn(U, d) and
    0.01 * randn(I, d), each cast to float32 (ExpoMF.py: initModel), from the legacy numpy stream seeded with the
    run's seed; mu0 = 0.01."""
    r = np.random.RandomState(int(g['seed']))
    nu, ni = len(g['user_names']), len(g['item_names'])
    r.rand(nu, d)
    r.rand(ni, d)
    theta = INIT_STD * r.randn(nu, d).astype(np.float32)
    beta = INIT_STD * r.randn(ni, d).astype(np.float32)
    return theta, beta, INIT_MU * np.ones(ni, dtype=np.float32)


def golden_csrs(g):
    """User- and item-major CSRs (rowptr int64, cols int32) of a golden run's training list, as the reference's
    binary csr_matrix X and X.T (ascending columns, duplicates once)."""
    users = {n: k for k, n in enumerate(g['user_names'].tolist())}
    items = {n: k for k, n in enumerate(g['item_names'].tolist())}
    pairs = {(users[u], items[i]) for u, i in zip(g['train_users'].tolist(), g['train_items'].tolist())}
    pu = np.array(sorted(pairs), dtype=np.int64).reshape(-1, 2)

    def csr(rows, cols, n):
        order = np.lexsort((cols, rows))
        rowptr = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(rows, minlength=n), out=rowptr[1:])
        return rowptr, cols[order].astype(np.int32)
    return csr(pu[:, 0], pu[:, 1], len(users)), csr(pu[:, 1], pu[:, 0], len(items))
