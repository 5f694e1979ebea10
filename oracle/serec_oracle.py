"""float64 numpy restatement of SERec (model/ranking/SERec.py of the reference), on CSR inputs.

SERec is ExpoMF (oracle/expomf_oracle.py: the posterior and the row solve are imported from there) with a prior per
(user, item) pair.  The reference holds that prior as a dense U x I matrix,
    mu = (a + A_sum + (s-1)*S_sum - 1) / (a + b + (s-1)*S_sum + U - 2),   A_sum = tile(A, [U, 1]),   S_sum = T.dot(A_sum)
with A the summed posteriors per item and T the 0/1 (user, followee) matrix of the cleaned social view.  Every row of
A_sum is A, so S_sum[u, i] = deg_u * A_i: the prior is a function of A (float64 [I]) and deg (int [U]).  `T.dot` forms
that product by adding A_i to itself deg_u times; `prior` offers both that repeated sum (form='sum', the reference's
bits, for golden comparisons) and the single product (form='product', what the kernel computes).

One epoch: every user against beta with mu[u, :], every item against the new theta with mu[:, i] -- or with mu[i, :]
when users and items are as many (the reference picks the branch with `mu.shape[1] == X.shape[0]`) -- then A from the
new tables and the OLD mu[u, i], 1 on the training entries.  The first epoch's mu is the uniform float32 0.01,
promoted to double.  Test infrastructure only: the product never imports this module.
"""
import numpy as np

from oracle import expomf_oracle as EO

LAM = 1e-5 / 0.01     # SERec.py: lam_theta = lam_beta = 1e-5, lam_y = 0.01, used as lam / lam_y
LAM_Y = 0.01
A_PRIOR, B_PRIOR, S_SOCIAL = 1.0, 99.0, 2.2
INIT_MU, INIT_STD = 0.01, 0.5
MU0 = float(np.float32(INIT_MU))


def social_sum(A, deg):
    """S = T.dot(tile(A)) for the rows with degrees deg: A added to itself deg times, in float64 (scipy's csr_matvecs
    order).  A: [I], deg: [n] -> [n, I]."""
    A = np.asarray(A, dtype=np.float64)
    deg = np.asarray(deg, dtype=np.int64)
    S = np.zeros((deg.shape[0], A.shape[0]))
    for k in range(int(deg.max()) if deg.size else 0):
        S[deg > k] += A
    return S


def prior(A, deg, n_users, form='product', a=A_PRIOR, b=B_PRIOR, s=S_SOCIAL):
    """mu[u, i] (float64 [len(deg), I]) for the users with degrees deg, in the reference's operand order."""
    A = np.asarray(A, dtype=np.float64)[None, :]
    if form == 'sum':
        S = social_sum(A[0], deg)
    else:
        S = np.asarray(deg, dtype=np.float64)[:, None] * A
    return (a + A + (s - 1) * S - 1) / (a + b + (s - 1) * S + n_users - 2)


def mu_matrix(A, deg, n_items, form='product'):
    """The whole U x I prior, or the uniform float32 mu0 (promoted to double) when A is None (the first epoch)."""
    if A is None:
        return np.full((len(deg), n_items), MU0)
    return prior(A, deg, len(deg), form)


def degrees(user_names, relation):
    """Each training user's number of followees in the cleaned social view (base/socialRecommender.py): relations
    whose follower or followee is not a training user are dropped; a repeated (follower, followee) pair counts once;
    a self-follow counts.  These are the row sums of SERec.py's T.  int32 [len(user_names)]."""
    ids = {n: k for k, n in enumerate(list(user_names))}
    followees = {}
    for u1, u2 in ((r[0], r[1]) for r in relation):
        followees.setdefault(u1, set()).add(u2)
    deg = np.zeros(len(ids), dtype=np.int32)
    for u1, fs in followees.items():
        if u1 in ids:
            deg[ids[u1]] = sum(1 for f in fs if f in ids)
    return deg


def solve_side(X, Z, rowptr, cols, M, lam=LAM, lam_y=LAM_Y, rows=None):
    """recompute_factors in place on X (rows rounded to X's dtype) against Z; row r uses the priors M[r] (one per row
    of Z).  Returns the number of rows left unchanged because their system was not positive definite."""
    failed = 0
    for r in (range(X.shape[0]) if rows is None else rows):
        x = EO.solve_row(X[r], Z, cols[rowptr[r]:rowptr[r + 1]], M[r], lam, lam_y)
        if x is None:
            failed += 1
        else:
            X[r] = x
    return failed


def asum_rows(X, Z, rowptr, cols, M, lam_y=LAM_Y, rows=None):
    """The summed posteriors of the rows of X (the items) against every row of Z (the users), as the item half of the
    engine computes them: sum_k A_k with A from x_r.z_k and M[r, k], 1 on row r's observed columns.  float64, one
    entry per row listed (default: all)."""
    Z64 = np.asarray(Z, dtype=np.float64)
    out = []
    for r in (range(X.shape[0]) if rows is None else rows):
        A = EO.exposure(Z64.dot(np.asarray(X[r], dtype=np.float64)), M[r], lam_y)
        A[np.asarray(cols[rowptr[r]:rowptr[r + 1]], dtype=np.int64)] = 1.0
        out.append(A.sum())
    return np.array(out, dtype=np.float64)


def epoch(theta, beta, A, deg, user_csr, item_csr, square_quirk=None, form='product', lam=LAM, lam_y=LAM_Y):
    """One epoch in place on theta and beta (float32 arrays) from the summed posteriors A (None: the first epoch).
    square_quirk: whether the item half reads mu[i, :]; None follows the reference (when users and items are as
    many).  Returns (the new A, the number of failed rows)."""
    n_users, n_items = theta.shape[0], beta.shape[0]
    M = mu_matrix(A, deg, n_items, form)
    failed = solve_side(theta, beta, user_csr[0], user_csr[1], M, lam, lam_y)
    if square_quirk is None:
        square_quirk = n_users == n_items
    failed += solve_side(beta, theta, item_csr[0], item_csr[1], M if square_quirk else M.T, lam, lam_y)
    return asum_rows(beta, theta, item_csr[0], item_csr[1], M.T, lam_y), failed


def initial_state(g, d):
    """theta0, beta0 of a golden run (float32): the base initModel's P / Q draws, then 0.5 * randn(U, d) and
    0.5 * randn(I, d), each cast to float32 (SERec.py: initModel), from the legacy numpy stream seeded with the run's
    seed.  The prior starts uniform (A = None)."""
    r = np.random.RandomState(int(g['seed']))
    nu, ni = len(g['user_names']), len(g['item_names'])
    r.rand(nu, d)
    r.rand(ni, d)
    theta = INIT_STD * r.randn(nu, d).astype(np.float32)
    beta = INIT_STD * r.randn(ni, d).astype(np.float32)
    return theta, beta
