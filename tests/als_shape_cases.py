"""Widths, row structures and float64 references for the ALS-family row solves of qrec_b200/csrc/als_kernels.cu: the
Gram, the WRMF row solve, the CoFactor item sweep and the exposure solve of ExpoMF and SERec.

Every one of them accumulates the upper triangle of its d x d system in 4x4 tiles (tiles_of(d) of them), NT = 1 or 3
tiles per thread (als_tiles_per_thread), and splits each stage of kStage = 32 staged rows over ngroups groups
(als_groups) that are reduced in group order.  Across d = 1..128 that gives 13 (NT, ngroups) classes; the widths below
reach both ends of each, every d mod 4 at both NT (the zero-filled padding columns of pad4), and 97..127, where warp
0's fourth substitution register is partly filled.  The builders reach the row lengths around each width's ngroups,
around one and two stages, a row longer than 1024 entries, more rows than the persistent grid holds at once, Gram
sizes around its 2048-row chunks, exposure tables around a stage, and CoFactor context lists around the same lengths.

Inputs are integers where that makes the system exact: |z| <= 4, ratings 1..5, ALPHA = 10, lambda = 1.  Every entry
of the Gram and of WRMF's A and b is then an integer far below 2^53, exact in float64 whatever the summation order,
so the Gram and the WRMF loss are compared bit for bit and a WRMF row's error comes from the Cholesky and the
substitutions alone.

A plain module, not collected: test_gpu_als_shape_matrix.py applies the references to the kernels and
test_als_shape_cases_cpu.py proves, without a GPU, that the tables reach every class and edge, that the references
agree with the oracles, that the device's own step source lies inside the bounds and that every defect lies outside."""
import functools
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import expomf_oracle as EO       # noqa: E402
from oracle import serec_oracle as SO        # noqa: E402

U32, U64 = 2.0 ** -24, 2.0 ** -53      # unit roundoff of fp32 and fp64

# ---------------------------------------------------------------------------------------------------------------------
# the tile layout (als_step.cuh; test_als_shape_cases_cpu.py checks this restatement against the header's own functions)
THREADS, STAGE, GRAM_CHUNK, MAX_D = 256, 32, 2048, 128


def pad4(d):
    return (d + 3) & ~3


def tiles_of(d):
    nb = pad4(d) // 4
    return nb * (nb + 1) // 2


def tiles_per_thread(d):
    return 1 if tiles_of(d) <= THREADS else 3


def groups(d):
    return min(tiles_per_thread(d) * THREADS // tiles_of(d), STAGE)


def tile_class(d):
    return tiles_per_thread(d), groups(d)


WIDTHS = (1, 2, 3, 4, 5, 12, 13, 16, 17, 20, 21, 24, 25, 28, 29, 32, 33, 36, 37, 40, 41, 48, 49, 60, 61,
          87, 88, 89, 90, 91, 92, 96, 97, 107, 108, 109, 125, 126, 127, 128)
# one width per class (its smallest) takes the 'many' structure as well, and the all-failing WRMF call
CLASS_WIDTHS = tuple(d for k, d in enumerate(WIDTHS) if all(tile_class(e) != tile_class(d) for e in WIDTHS[:k]))

SMS = 132              # an H100 SXM
MAX_PER_SM = 3         # __launch_bounds__ of the NT = 1 row solves; NT = 3 and the sweep allow fewer
MANY = 420             # rows of the 'many' structure: more than SMS * MAX_PER_SM CTAs take at once
LONG = 1100            # a row longer than 1024 entries
ALPHA, LAM = 10.0, 1.0
LAM_Y = 1.0            # the exposure solves' lam_y: posteriors of the small old rows near sqrt(1/2 pi), so they matter
UNNAMED = 3            # rows of every solve case that its row order leaves out


def row_lengths(d):
    g = groups(d)
    return sorted({0, 1, g - 1, g, g + 1, 31, 32, 33, 63, 64, 65, LONG})


GRAM_SIZES = (0, 1, 31, 32, 33, 2047, 2048, 2049, 3 * 2048 + 17)
EXPO_M = {'tails': 40, 'many': 3}      # exposure tables of 32m, 32m + 1 or 32m + 31 rows


def expo_rows(d, structure):
    m = EXPO_M[structure]
    return (32 * m, 32 * m + 1, 32 * m + 31)[WIDTHS.index(d) % 3]


def _ints(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float64)


def _csr(rng, lengths, n_cols):
    rowptr = np.zeros(len(lengths) + 1, np.int64)
    rowptr[1:] = np.cumsum(lengths)
    cols = np.concatenate([rng.choice(n_cols, int(k), replace=False) for k in lengths] + [np.zeros(0, int)])
    return rowptr, cols.astype(np.int32)


def _order(rng, lengths):
    """Rows longest first (als_row_order) without UNNAMED rows that have entries."""
    busy = np.nonzero(np.asarray(lengths) > 0)[0]
    skip = rng.choice(busy, UNNAMED, replace=False)
    named = np.setdiff1d(np.arange(len(lengths)), skip)
    return named[np.argsort(-np.asarray(lengths)[named], kind='stable')].astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# builders
@functools.lru_cache(maxsize=None)
def gram_case(d, n):
    return _ints(np.random.default_rng([1, d, n]), (n, d))


@functools.lru_cache(maxsize=None)
def solve_case(d, structure):
    """A WRMF half: X (integer old rows), Z, the rating CSR (integer ratings) and a row order.  'tails': one row of
    every row_lengths(d) against 1200 rows of Z; 'many': MANY rows of 0..40 entries."""
    rng = np.random.default_rng([2, d, ('tails', 'many').index(structure)])
    if structure == 'tails':
        lengths, n_z = rng.permutation(row_lengths(d)), 1200
    else:
        lengths, n_z = rng.integers(0, 41, MANY), 200
    rowptr, cols = _csr(rng, lengths, n_z)
    return dict(X=_ints(rng, (len(lengths), d)), Z=_ints(rng, (n_z, d)), rowptr=rowptr, cols=cols,
                vals=rng.integers(1, 6, len(cols)).astype(np.float64), order=_order(rng, lengths))


@functools.lru_cache(maxsize=None)
def exposure_case(d, structure):
    """An exposure half: X (small old rows, so that the posteriors matter), Z (integers, expo_rows(d) rows), the
    observed CSR, a row order, ExpoMF priors by column and by row, and SERec's summed posteriors and degrees for
    X's rows and for Z's rows (degree 0 among them)."""
    rng = np.random.default_rng([3, d, ('tails', 'many').index(structure)])
    n_z = expo_rows(d, structure)
    lengths = rng.permutation(row_lengths(d)) if structure == 'tails' else rng.integers(0, 41, MANY)
    rowptr, cols = _csr(rng, lengths, n_z)
    n = len(lengths)
    f32 = np.float32
    X = (rng.integers(-4, 5, (n, d)) / (16.0 * d)).astype(f32)
    deg = lambda k: (rng.integers(0, 40, k) * (rng.random(k) < 0.6)).astype(np.int32)   # noqa: E731
    return dict(X=X, Z=_ints(rng, (n_z, d)).astype(f32), rowptr=rowptr, cols=cols, order=_order(rng, lengths),
                mu_z=rng.uniform(0.005, 0.05, n_z).astype(f32), mu_x=rng.uniform(0.005, 0.05, n).astype(f32),
                asum_x=rng.uniform(0.0, 20.0, n), asum_z=rng.uniform(0.0, 20.0, n_z), deg_x=deg(n), deg_z=deg(n_z))


def context_lengths(d):
    return sorted({0, 1, groups(d), 31, 32, 33, 65})


@functools.lru_cache(maxsize=None)
def cofactor_case(d, dtype):
    """An item sweep: a symmetric SPPMI made of stars -- a centre with k contexts, each a leaf with one context, for
    every k of context_lengths(d) above 0 -- and three items without contexts, ids shuffled so that contexts lie on
    both sides of their item; every item's user list has one of the same lengths."""
    rng = np.random.default_rng([4, d, 0 if dtype == 'float32' else 1])
    edges, n = [], 0
    for k in context_lengths(d):
        if k == 0:
            continue
        edges += [(n, n + 1 + j) for j in range(k)]
        n += k + 1
    n_items = n + 3
    perm = rng.permutation(n_items)
    e = np.array([(perm[a], perm[b]) for a, b in edges])
    val = rng.uniform(0.1, 1.0, len(e))             # no eighths: no right-hand side cancels exactly to 0
    rows, cols, vals = np.concatenate([e[:, 0], e[:, 1]]), np.concatenate([e[:, 1], e[:, 0]]), np.tile(val, 2)
    srt = np.lexsort((cols, rows))
    srp = np.zeros(n_items + 1, np.int64)
    srp[1:] = np.cumsum(np.bincount(rows, minlength=n_items))
    n_users = 80
    ulen = rng.permutation(np.resize(context_lengths(d), n_items))
    irp, icol = _csr(rng, ulen, n_users)
    dt = np.dtype(dtype)
    return dict(X=_ints(rng, (n_users, d)).astype(dt), Y=_ints(rng, (n_items, d)).astype(dt),
                G=_ints(rng, (n_items, d)).astype(dt), w=(rng.integers(-4, 5, n_items) / 8).astype(dt),
                c=(rng.integers(-4, 5, n_items) / 8).astype(dt),
                item_csr=(irp, icol, rng.integers(1, 6, len(icol)).astype(dt)),
                sppmi=(srp, cols[srt].astype(np.int32), vals[srt].astype(dt)))


# ---------------------------------------------------------------------------------------------------------------------
# defects: each reference below can be rebuilt with one of them, and the bounds must tell every one of them apart
DEFECTS = ('drop_last', 'column', 'group', 'lambda')
#   drop_last -- the last staged entry of every row is dropped (the exposure dense pass: the last row of Z)
#   column    -- column d-1 of every staged row reads 0
#   group     -- the tile sums leave out the entries of group ngroups-1 of every stage (ngroups = 1: the last stage)
#   lambda    -- lambda is left off the last diagonal element


def applies(defect, lengths, d):
    """Whether a defect touches a case whose staged lists have these lengths: 'group' only where some stage has an
    entry in group ngroups-1 (or, at ngroups = 1, some list is not empty)."""
    return defect != 'group' or any(tile_weights(n, d, defect).min(initial=1) == 0 for n in lengths)


def tile_weights(n, d, defect):
    """1/0 per staged entry of an n-entry list in the tile sums under `defect`."""
    keep = np.ones(n)
    if defect == 'group' and n:
        g, k = groups(d), np.arange(n)
        keep[(k % STAGE) % g == g - 1 if g > 1 else k >= STAGE * ((n - 1) // STAGE)] = 0
    return keep


def staged(Z, defect):
    Z = np.array(Z, np.float64)
    if defect == 'column':
        Z[:, -1] = 0
    return Z


def entries(cols, *per_entry, defect=None):
    if defect == 'drop_last' and len(cols):
        return (cols[:-1],) + tuple(v[:-1] for v in per_entry)
    return (cols,) + per_entry


def kappa(A):
    return float(np.abs(A).sum(1).max() * np.abs(np.linalg.inv(A)).sum(1).max())


def refined_solve(A, b):
    """np.linalg.solve plus one step of iterative refinement with the residual in long double: A and b are exact
    integers, so the residual carries long double's rounding alone, 2^-11 of a double's."""
    x = np.linalg.solve(A, b)
    r = b.astype(np.longdouble) - A.astype(np.longdouble) @ x.astype(np.longdouble)
    return x + np.linalg.solve(A, r.astype(np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# references
def solve_systems(c, defect=None):
    """WRMF's (A, b) of every row in c['order'] (als_solve_rows_kernel: A = (G + S) + lambda I)."""
    Z = np.asarray(c['Z'], np.float64)
    d = Z.shape[1]
    G = Z.T @ Z
    out = []
    for r in c['order']:
        a, e = c['rowptr'][r], c['rowptr'][r + 1]
        cols, vals = entries(c['cols'][a:e], c['vals'][a:e], defect=defect)
        z = staged(Z[cols], defect)
        w = ALPHA * vals
        A = G + (z * (w * tile_weights(len(cols), d, defect))[:, None]).T @ z + LAM * np.eye(d)
        if defect == 'lambda':
            A[d - 1, d - 1] -= LAM
        out.append((A, ((1.0 + w)[:, None] * z).sum(0)))
    return out


@functools.lru_cache(maxsize=None)
def solve_reference(d, structure, defect=None):
    """(x [rows of the order], kappa per row): the refined float64 solutions."""
    c = solve_case(d, structure)
    sys_ = solve_systems(c, defect)
    x = np.array([refined_solve(A, b) for A, b in sys_]).reshape(len(sys_), d)
    return x, (np.array([kappa(A) for A, _ in sys_]) if defect is None else None)


def solve_loss(c):
    """sum (1 - x_old.z)^2 over the order's entries, in integers (exact)."""
    X, Z = np.asarray(c['X']).astype(np.int64), np.asarray(c['Z']).astype(np.int64)
    tot = 0
    for r in c['order']:
        z = Z[c['cols'][c['rowptr'][r]:c['rowptr'][r + 1]]]
        tot += int(((1 - z @ X[r]) ** 2).sum())
    return tot


def exposure_prior(c, kind, asum_given, row_is_user=True):
    """The prior matrix M [rows of X, rows of Z] of a call: ExpoMF by column ('expomf_user', mu_z) or by row
    ('expomf_item', mu_x); SERec ('serec') from the case's sums and degrees (or the uniform MU0) with X's rows the
    users or the items."""
    n, n_z = len(c['X']), len(c['Z'])
    if kind == 'expomf_user':
        return np.broadcast_to(c['mu_z'].astype(np.float64), (n, n_z))
    if kind == 'expomf_item':
        return np.broadcast_to(c['mu_x'].astype(np.float64)[:, None], (n, n_z))
    if row_is_user:
        return SO.mu_matrix(c['asum_z'] if asum_given else None, c['deg_x'], n_z)
    return SO.mu_matrix(c['asum_x'] if asum_given else None, c['deg_z'], n).T


def exposure_row(x_old, Z, cols, prior, lam, lam_y, defect=None):
    """(B, b) of one exposure row (exposure_solve_rows_kernel): a dense pass over every row of Z weighted by its
    posterior, a correction pass lifting the observed entries to 1, b the sum of the observed rows."""
    d, n_z = Z.shape[1], Z.shape[0]
    Zs = staged(Z, defect)
    A = np.broadcast_to(EO.exposure(Zs @ np.asarray(x_old, np.float64), prior, lam_y), (n_z,)).copy()
    wd = A * tile_weights(n_z, d, defect)
    if defect == 'drop_last':
        wd[-1] = 0
    cols = np.asarray(cols, np.int64)
    wc = (1.0 - A[cols]) * tile_weights(len(cols), d, defect)
    B = (Zs.T * wd) @ Zs + (Zs[cols].T * wc) @ Zs[cols] + lam * np.eye(d)
    if defect == 'lambda':
        B[d - 1, d - 1] -= lam
    return B, Zs[cols].sum(0)


def exposure_reference(c, M, lam, lam_y, defect=None):
    """(x [rows of the order] float64, kappa per row) of an exposure half with priors M."""
    Z = np.asarray(c['Z'], np.float64)
    xs, ks = [], []
    for r in c['order']:
        B, b = exposure_row(c['X'][r], Z, c['cols'][c['rowptr'][r]:c['rowptr'][r + 1]], M[r], lam, lam_y, defect)
        xs.append(np.linalg.solve(B, b))
        ks.append(kappa(B) if defect is None else np.nan)
    return np.array(xs).reshape(len(xs), Z.shape[1]), np.array(ks)


def exposure_sums(c, X_new, M_out, lam_y, defect=None):
    """The fused pass of the item half: sum_k A_k of each row of the order with its new value and the out priors,
    1 on its observed columns (serec_oracle.asum_rows, with the defects of the dense pass)."""
    Z = staged(c['Z'], defect)
    out = []
    for r in c['order']:
        A = np.broadcast_to(EO.exposure(Z @ np.asarray(X_new[r], np.float64), M_out[r], lam_y), (len(Z),)).copy()
        dense = A.copy()
        if defect == 'drop_last':
            dense[-1] = 0
        cols = np.asarray(c['cols'][c['rowptr'][r]:c['rowptr'][r + 1]], np.int64)
        out.append(dense.sum() + (1.0 - A[cols]).sum())        # the dense pass, then the lift of the observed rows
    return np.array(out)


def cofactor_reference(c, lam, gamma, defect=None):
    """The in-order item sweep (cofactor_oracle.item_sweep) on copies of the case's tables, rows stored in the case's
    dtype; with the defects of the staging, the tile sums and the diagonal.  Returns (Y, G, w, c, kappa_Y, kappa_G,
    scale_w, scale_c): kappa per item (nan where an item has no G system) and the mean absolute term of w's and c's
    sums (0 without contexts)."""
    Y, G, w, cc = (np.array(c[k], copy=True) for k in ('Y', 'G', 'w', 'c'))
    X = np.asarray(c['X'], np.float64)
    irp, icol, ival = c['item_csr']
    srp, scol, sval = c['sppmi']
    d = X.shape[1]
    XtX, eye = X.T @ X, np.eye(d)
    kY, kG = np.full(len(Y), np.nan), np.full(len(Y), np.nan)
    sw, sc = np.zeros(len(Y)), np.zeros(len(Y))
    for i in range(len(Y)):
        u, v = entries(icol[irp[i]:irp[i + 1]], np.asarray(ival[irp[i]:irp[i + 1]], np.float64), defect=defect)
        ctx, m = entries(scol[srp[i]:srp[i + 1]], np.asarray(sval[srp[i]:srp[i + 1]], np.float64), defect=defect)
        xu = staged(X[u], defect)
        gam, bet = staged(G[ctx], defect), staged(Y[ctx], defect)
        w_c, c_c = np.asarray(w[ctx], np.float64), np.asarray(cc[ctx], np.float64)
        w_i, c_i = float(w[i]), float(cc[i])
        y_old, g_old = np.array(Y[i], np.float64), np.array(G[i], np.float64)
        tu, tc = tile_weights(len(u), d, defect), tile_weights(len(ctx), d, defect)
        A = XtX + (xu * (ALPHA * v * tu)[:, None]).T @ xu + lam * eye + (gam * tc[:, None]).T @ gam
        if defect == 'lambda':
            A[d - 1, d - 1] -= lam
        b = ((1.0 + ALPHA * v)[:, None] * xu).sum(0) + (((m - w_i) - c_c)[:, None] * gam).sum(0)
        Y[i] = np.linalg.solve(A, b)
        kY[i] = kappa(A) if defect is None else np.nan
        if len(scol[srp[i]:srp[i + 1]]):
            B = (bet * tc[:, None]).T @ bet + gamma * eye
            G[i] = np.linalg.solve(B, (((m - w_c) - c_i)[:, None] * bet).sum(0))
            kG[i] = kappa(B) if defect is None else np.nan
            n_ctx = srp[i + 1] - srp[i]
            w[i] = ((m - gam @ y_old) - c_c).sum() / n_ctx
            cc[i] = ((m - bet @ g_old) - w_c).sum() / n_ctx
            sw[i] = (np.abs(m) + np.abs(gam) @ np.abs(y_old) + np.abs(c_c)).sum() / n_ctx
            sc[i] = (np.abs(m) + np.abs(bet) @ np.abs(g_old) + np.abs(w_c)).sum() / n_ctx
    return Y, G, w, cc, kY, kG, sw, sc


# ---------------------------------------------------------------------------------------------------------------------
# error measures and bounds
def row_errors(got, ref):
    """|got - ref|_inf / |ref|_inf per row (rows of ref that are 0 must be exactly 0)."""
    err = np.abs(np.asarray(got, np.float64) - ref).max(1)
    scale = np.abs(ref).max(1)
    return np.where(scale > 0, err / np.where(scale > 0, scale, 1.0), np.where(err > 0, np.inf, 0.0))


def solve_units(d, kap, f32, c=1.0):
    """The per-row unit c d 2^-53 kappa_inf(A), plus 2^-24 for float32 rows (their rounding when stored)."""
    return c * d * U64 * np.asarray(kap) + (U32 if f32 else 0.0)


def cofactor_units(c, ref, f32):
    """Per-item units of the sweep's outputs, where A is not exact: its float64 sums over the item's n contexts are
    reordered as well, so Y and G rows take (d + n) 2^-53 kappa_inf(A) (+ 2^-24), and w and c, means of n terms
    of d-long dots, (d + n) 2^-53 (+ 2^-24) times their mean absolute term."""
    d = c['X'].shape[1]
    n = np.diff(c['sppmi'][0])
    kY, kG, sw, sc = ref[4:]
    extra = U32 if f32 else 0.0
    return ((d + n) * U64 * kY + extra, (d + n) * U64 * np.nan_to_num(kG) + extra,
            ((d + n) * U64 + extra) * sw, ((d + n) * U64 + extra) * sc)


# A solved row with an exact A and b lies within solve_units(d, kappa, f32, C_SOLVE) of the refined solution: the
# Cholesky and the substitutions (x = b / a at d = 1 already takes four roundings: sqrt, 1/, and two products).
C_SOLVE = 8.0
# The other families' bounds, in the units of solve_units (Y, G and X rows), cofactor_units (w, c), 2^-24 of |mu|
# (ExpoMF's fused prior) and n_z 2^-53 of |A| (SERec's fused sums): about 3 x the largest ratio observed over the
# family's cases on an H100 80GB HBM3 (700 W power limit), given beside each.  CoFactor's float64 G rows are far from
# their own system's rounding, and float64 Y rows at small d from theirs: the rows of earlier items of the same sweep
# carry their own error into A and b.
BOUNDS = {
    'cofactor_f64': {'Y': 85.0, 'G': 750.0, 'w': 4.5, 'c': 7.0},       # 27.8, 244, 1.4, 2.2
    'cofactor_f32': {'Y': 3.5, 'G': 6.0, 'w': 0.15, 'c': 0.15},        # 1.04, 1.98, 0.035, 0 (bit-equal)
    'expomf': {'X': 3.0, 'mu_out': 3.0},                               # 0.98, 0.97
    'serec': {'X': 3.0, 'asum_out': 0.15},                             # 1.0, 0.051
}
TEETH = 10.0           # every defective reference must lie at least this many bounds away


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def worst(errors, units):
    return float(np.max(np.asarray(errors) / np.asarray(units))) if len(errors) else 0.0


def judge(name, bounds, outputs):
    """outputs: {output: (observed, {defect: distance})} in the units of `bounds`; defects that do not apply are left
    out.  Prints both over the bound and asserts that the kernel is inside every bound and every defect at least
    TEETH bounds outside it."""
    line = []
    for key, (obs, bad) in outputs.items():
        near = min(bad.values()) if bad else math.inf
        line.append('%s %.3g/%.3g' % (key, obs / bounds[key], near / bounds[key]))
    print('\n%s observed/bound, nearest defect/bound: %s' % (name, ', '.join(line)))
    for key, (obs, bad) in outputs.items():
        assert obs <= bounds[key], '%s: %s off by %.4g, bound %.4g' % (name, key, obs, bounds[key])
        for defect, dist in bad.items():
            assert dist >= TEETH * bounds[key], '%s: the %s bound cannot tell %s (%.4g)' % (name, key, defect, dist)
