"""Widths, row structures and float64 references for the row-parallel kernels behind the lane-group dispatch
(qrec_b200/csrc/lane_shape.h) outside the user-major BPR epoch: the SpMM family, K3, the staged BPR step, the MF batch
and ordered steps and the SVD++ user-major epoch.

A row kernel runs one lane group of LPR lanes per row, VPL float4 slices per lane; the parity kernels run one warp per
entry, E elements per lane.  Each launcher is compiled for every shape its width cap allows, and each shape exists with
all lanes busy (d = 4 LPR VPL, d = 32 E) and with idle lanes.  The widths below reach all of them, and the builders
reach the branches where a mask like `l + v*LPR < nvec` or `(t+q) < m` or a group-masked shuffle can be wrong at one
shape and right at another: ragged row lengths around the lane-group size and the gather batch, rows longer than a
balanced chunk and than one scatter pass, -1 padding, empty users inside a row order, and launches with more rows or
entries than lane groups.

A plain module, not collected: test_gpu_row_shape_matrix.py applies the references to the kernels and
test_row_shape_cases_cpu.py proves, without a GPU, that the tables reach every shape and branch and that the new
references agree with the existing oracles."""
import math

import numpy as np

U32, U64 = 2.0 ** -24, 2.0 ** -53      # unit roundoff of fp32 and fp64

# ---------------------------------------------------------------------------------------------------------------------
# widths per launcher cap
WIDTHS_256 = (4, 8, 12, 16, 20, 28, 32, 48, 52, 64, 100, 128, 132, 200, 256)
WIDTHS_128 = tuple(d for d in WIDTHS_256 if d <= 128)
# the warp-per-entry parity kernels: E = 1, 2, 4, 8 elements per lane, each with all lanes busy (d = 32 E) and idle
WIDTHS_PARITY = (1, 31, 32, 33, 64, 65, 100, 128, 129, 200, 256)

# launcher -> width cap (128 or 256) or 'parity'
LAUNCHERS = {
    'spmm_balanced': 256,       # spmm_csr_balanced_kernel<LPR, VPL, 1024>
    'spmm_rowsplit': 256,       # spmm_csr_kernel<LPR, VPL>; d = 64 takes spmm_csr_d64_kernel
    'spmm_scatter_rows': 128,   # spmm_scatter_rows_kernel<LPR>
    'spmm_rows': 128,           # spmm_list_rows_kernel<LPR>
    'k3': 256,                  # bpr_grad_scatter_kernel<LPR, VPL, UNROLL, MODE>
    'bpr_staged': 128,          # bpr_sgd_staged_kernel<LPR>
    'mf_batch': 128,            # mf_sgd_batch_kernel<LPR, KIND, 4>
    'mf_ordered': 'parity',     # mf_sgd_ordered_kernel<T, E, KIND>
    'svdpp_usermajor': 128,     # svdpp_usermajor_kernel<LPR>
}


def widths(launcher):
    cap = LAUNCHERS[launcher]
    return WIDTHS_PARITY if cap == 'parity' else WIDTHS_256 if cap == 256 else WIDTHS_128


def row_shape(d, max_d):
    """lane_shape.h: (LPR, VPL) of a row of d floats under with_row_shape<max_d>."""
    nvec = d // 4
    lpr = 4 if nvec <= 4 else 8 if nvec <= 8 else 16 if nvec <= 16 else 32
    return (32, 2) if max_d > 128 and nvec > 32 else (lpr, 1)


def lane_elems(d):
    e = (d + 31) // 32
    return 1 if e <= 1 else 2 if e <= 2 else 4 if e <= 4 else 8


# ---------------------------------------------------------------------------------------------------------------------
# kernel constants the structures are built around
CHUNK = 1024           # spmm_csr_balanced_kernel: QN non-zeros per lane group
SLICE, PASS = 64, 64   # spmm_scatter_rows_kernel: edges per slice, slices per pass over a source row (4096 edges)
K_PREFETCH = 4         # svdpp_kernels.cu: kPrefetch
SMS = 132              # an H100 SXM; the launch sizing (capped_grid) allows 8 CTAs of 256 threads per SM


def lane_groups(lpr, blocks_per_sm=8):
    """Lane groups of a launch capped at blocks_per_sm CTAs of 256 threads per SM."""
    return SMS * blocks_per_sm * 256 // lpr


def rowsplit_gather(vpl):
    """spmm_csr_kernel: gathered X rows in flight per lane (G)."""
    return 8 if vpl == 1 else 4


def row_lengths(lpr):
    """Every length 0 .. 2 LPR + 1 (0, 1, LPR - 1, LPR, LPR + 1 and each multiple of the gather batch and of LPR up to
    2 LPR + 1), and lengths around two row-split gather batches, the list kernel's 4 x 32/LPR batches and the scatter
    kernel's 64-edge slices."""
    return sorted(set(range(2 * lpr + 2)) | {15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129})


LONG_ROWS = (1023, 1024, 1025, 2049, 4095, 4096, 4097, 2 * SLICE * PASS + 3, 12_289)


def _csr(rng, lengths, n_cols):
    rowptr = np.zeros(len(lengths) + 1, np.int64)
    rowptr[1:] = np.cumsum(lengths)
    cols = np.concatenate([np.sort(rng.choice(n_cols, int(k), replace=False)) for k in lengths] + [np.zeros(0, int)])
    vals = rng.standard_normal(len(cols)).astype(np.float32)
    return rowptr, cols.astype(np.int32), vals


def spmm_case(launcher, d, structure):
    """A CSR matrix A (rowptr int64, cols int32, vals fp32), X, the accumulated table acc0 and, for the row-list
    kernels, the row list (int32 with -1 padding).  structure: 'tails' (row_lengths of the width's lane group, each
    many times, shuffled, with empty rows at both ends) or 'long' (rows longer than a balanced chunk and than one
    scatter pass among short rows, empty rows between them)."""
    rng = np.random.default_rng([list(LAUNCHERS).index(launcher), d, ('tails', 'long').index(structure)])
    lpr = row_shape(d, LAUNCHERS[launcher])[0]
    if structure == 'tails':
        lengths = rng.permutation(np.tile(row_lengths(lpr), -(-1500 // len(row_lengths(lpr)))))
        lengths = np.concatenate([[0, 0], lengths, [0, 0]])
        n_cols = 600
    else:
        lengths = rng.integers(0, 41, 300)
        at = np.sort(rng.choice(np.arange(10, 290), len(LONG_ROWS), replace=False))
        lengths[at] = LONG_ROWS
        lengths[at + 1] = 0
        lengths[-3:] = 0
        n_cols = 13_000
    rowptr, cols, vals = _csr(rng, lengths, n_cols)
    n_rows = len(lengths)
    if launcher == 'spmm_scatter_rows':          # A holds the source rows' edge lists: Y (n_cols rows) = A[listed]^T X
        X = rng.standard_normal((n_rows, d)).astype(np.float32)
        acc0 = rng.standard_normal((n_cols, d)).astype(np.float32)
    else:
        X = rng.standard_normal((n_cols, d)).astype(np.float32)
        acc0 = rng.standard_normal((n_rows, d)).astype(np.float32)
    rows = None
    if launcher in ('spmm_scatter_rows', 'spmm_rows'):
        # distinct rows, sorted, every fifth slot -1 padding (graphRecommender.sorted_unique_padded's output has that form)
        listed = np.sort(rng.choice(n_rows, n_rows * 3 // 4 if structure == 'tails' else n_rows - 40, replace=False))
        if structure == 'long':
            listed = np.union1d(listed, np.nonzero(lengths > CHUNK)[0])
        rows = np.full(len(listed) + len(listed) // 4, -1, np.int32)
        rows[np.sort(rng.choice(len(rows), len(listed), replace=False))] = listed
    return dict(rowptr=rowptr, cols=cols, vals=vals, X=X, acc0=acc0, rows=rows, n_rows=n_rows, n_cols=n_cols)


def csr_matrix(c, drop_last=False):
    """The case's matrix in float64; drop_last removes the last entry of every row (the defect the bounds must see)."""
    from scipy import sparse
    rowptr, cols, vals = c['rowptr'], c['cols'], c['vals'].astype(np.float64)
    if drop_last:
        keep = np.ones(len(cols), bool)
        ends = rowptr[1:][np.diff(rowptr) > 0] - 1
        keep[ends] = False
        row = np.repeat(np.arange(c['n_rows']), np.diff(rowptr))
        return sparse.csr_matrix((vals[keep], (row[keep], cols[keep])), shape=(c['n_rows'], c['n_cols']))
    return sparse.csr_matrix((vals, cols, rowptr), shape=(c['n_rows'], c['n_cols']))


def spmm_reference(launcher, c, drop_last=False):
    """(Y, |terms| summed per element) in float64 for the whole output of the launcher; rows a row-list launch does not
    produce are None-free: spmm_rows returns only the listed rows (in list order, -1 dropped)."""
    A = csr_matrix(c, drop_last)
    X = c['X'].astype(np.float64)
    if launcher == 'spmm_scatter_rows':
        listed = c['rows'][c['rows'] >= 0]
        B = A[listed]
        return np.asarray((B.T @ X[listed])), np.asarray(abs(B).T @ np.abs(X[listed]))
    if launcher == 'spmm_rows':
        listed = c['rows'][c['rows'] >= 0]
        return np.asarray(A[listed] @ X), np.asarray(abs(A[listed]) @ np.abs(X))
    return np.asarray(A @ X), np.asarray(abs(A) @ np.abs(X))


# ---------------------------------------------------------------------------------------------------------------------
# K3: the BPR gradient scatter of the graph models
K3_ENTRIES = ('grad', 'scaled', 'partial_scores', 'grad_from_scores')   # MODE 0, MODE 0 with y_scale, MODE 1, MODE 2
K3_SIZES = {'batch': 1237, 'short': 5}                                     # triples; neither a multiple of a warp


def k3_case(d, structure):
    """Distinct users and distinct items across the batch (no row is scattered to twice), one triple in ten with
    u = -1 (another rank's triple, skipped), a per-triple score scale and given full scores."""
    n = K3_SIZES[structure]
    rng = np.random.default_rng([30, d, n])
    nu, ni = n + 20, 2 * n + 30
    U = (rng.standard_normal((nu, d)) * 0.3).astype(np.float32)
    V = (rng.standard_normal((ni, d)) * 0.3).astype(np.float32)
    u = rng.permutation(nu)[:n].astype(np.int32)
    ij = rng.permutation(ni)[:2 * n].astype(np.int32)
    i, j = ij[:n].copy(), ij[n:].copy()
    u[rng.random(n) < 0.1] = -1
    u[n // 2] = -1
    gU0 = rng.standard_normal((nu, d)).astype(np.float32)
    gV0 = rng.standard_normal((ni, d)).astype(np.float32)
    y_scale = rng.uniform(0.3, 1.0, n).astype(np.float32)
    y_full = (rng.standard_normal(n) * 2).astype(np.float32)
    return dict(U=U, V=V, u=u, i=i, j=j, gU0=gU0, gV0=gV0, y_scale=y_scale, y_full=y_full)


def k3_reference(U, V, u, i, j, eps, reg, entry, y_scale=None, y_full=None, log_weight=1.0):
    """float64 restatement of bpr_grad_scatter_kernel's four entries over the triples with u >= 0 (util/loss.py:3-6 +
    the batch L2 term, LightGCN.py:28-30).  Returns (loss, gU, gV, y): grad -- loss and gradients; scaled -- the score
    of triple k is y_scale[k] y_k inside the -ln term; partial_scores -- y_k (0 for skipped triples) and the L2 term
    only; grad_from_scores -- gradients with y_full in place of the tables' score, loss = log_weight sum -ln(s + eps)."""
    ok = u >= 0
    uu, ii, jj = u[ok], i[ok], j[ok]
    pu, pi, pj = (T[x].astype(np.float64) for T, x in ((U, uu), (V, ii), (V, jj)))
    y = (pu * pi).sum(1) - (pu * pj).sum(1)
    l2 = reg * 0.5 * ((pu * pu).sum() + (pi * pi).sum() + (pj * pj).sum())
    if entry == 'partial_scores':
        y_out = np.zeros(len(u))
        y_out[ok] = y
        return float(l2), None, None, y_out
    c = np.ones(len(uu))
    if entry == 'scaled':
        c = y_scale[ok].astype(np.float64)
    if entry == 'grad_from_scores':
        y = y_full[ok].astype(np.float64)
    s = 1.0 / (1.0 + np.exp(-c * y))
    gy = (-(s * (1.0 - s) / (s + eps)) * c)[:, None]
    loss = (log_weight * -np.log(s + eps).sum()) if entry == 'grad_from_scores' else (-np.log(s + eps).sum() + l2)
    gU = np.zeros(U.shape)
    gV = np.zeros(V.shape)
    np.add.at(gU, uu, gy * (pi - pj) + reg * pu)
    np.add.at(gV, ii, gy * pu + reg * pi)
    np.add.at(gV, jj, -gy * pu + reg * pj)
    return float(loss), gU, gV, None


# ---------------------------------------------------------------------------------------------------------------------
# the staged BPR step (row-sharded item table)
def staged_groups(lpr):
    return lane_groups(lpr)


def staged_case(d, structure):
    """Distinct users; the rows of i and j at distinct positions of the staging buffer R, which has rows no triple
    names.  'ragged': 3001 triples; 'grid_stride': more triples than the launch has lane groups."""
    lpr = row_shape(d, 128)[0]
    n = 3001 if structure == 'ragged' else staged_groups(lpr) + 777
    rng = np.random.default_rng([40, d, n])
    nu, nr = n + 50, 2 * n + 13
    P = (rng.random((nu, d)) / 3).astype(np.float32)
    R = (rng.random((nr, d)) / 3).astype(np.float32)
    D0 = rng.standard_normal((nr, d)).astype(np.float32)
    u = rng.permutation(nu)[:n].astype(np.int32)
    pos = rng.permutation(nr)[:2 * n].astype(np.int32)
    return dict(P=P, R=R, D0=D0, u=u, pos_i=pos[:n].copy(), pos_j=pos[n:].copy())


def staged_reference(P, R, D, u, pos_i, pos_j, lr, reg_u, reg_i):
    """float64 BPR.py:45-53 on staged rows, the users distinct: qi = R[pos_i], qj = R[pos_j];
        x = p.qi - p.qj;  s = 1/(1+exp(-x));  g = lr (1 - s)
        pn = p + g (qi - qj);  qin = qi + g pn;  qjn = qj - g pn
        P[u] = pn - lr regU pn;  D[pos_i] = (qin - lr regI qin) - qi;  D[pos_j] = (qjn - lr regI qjn) - qj
    P is updated in place and the item deltas are written (not added) to D.  Returns (P, D, sum -ln s)."""
    P, D = P.astype(np.float64), D.astype(np.float64)
    p, qi, qj = P[u], R[pos_i].astype(np.float64), R[pos_j].astype(np.float64)
    x = (p * qi).sum(1) - (p * qj).sum(1)
    s = 1.0 / (1.0 + np.exp(-x))
    g = (lr * (1.0 - s))[:, None]
    pn = p + g * (qi - qj)
    qin, qjn = qi + g * pn, qj - g * pn
    P[u] = pn - lr * reg_u * pn
    D[pos_i] = (qin - lr * reg_i * qin) - qi
    D[pos_j] = (qjn - lr * reg_i * qjn) - qj
    return P, D, float(-np.log(s).sum())


# ---------------------------------------------------------------------------------------------------------------------
# the MF step (BasicMF / PMF / SVD)
PAD = 2                # zero padding columns at the end of the MF batch and SVD++ tables


def mf_batch_case(d, structure):
    """Distinct users and distinct items in the launch (Jacobi reading = sequential reading), the last PAD columns
    zero.  'ragged': 1237 entries over the full grid; 'windowed': 3001 entries through a grid that max_inflight
    bounds to one block, so that every lane group takes many grid-stride rounds."""
    n, window = (1237, 0) if structure == 'ragged' else (3001, 100)
    rng = np.random.default_rng([50, d, n])
    nu, ni = n + 40, n + 60
    P = (rng.random((nu, d)) / 3).astype(np.float32)
    Q = (rng.random((ni, d)) / 3).astype(np.float32)
    P[:, d - PAD:] = 0
    Q[:, d - PAD:] = 0
    u = rng.permutation(nu)[:n].astype(np.int32)
    i = rng.permutation(ni)[:n].astype(np.int32)
    r = (rng.integers(1, 9, n) / 2.0).astype(np.float32)
    Bu, Bi = (rng.random(nu) / 5).astype(np.float32), (rng.random(ni) / 5).astype(np.float32)
    return dict(P=P, Q=Q, u=u, i=i, r=r, Bu=Bu, Bi=Bi, max_inflight=window)


def mf_batch_groups(d, max_inflight):
    """Lane groups of qrec_mf_sgd_batch_f32's launch when max_inflight bounds it (4 entries in flight per group)."""
    lpr = row_shape(d, 128)[0]
    per_block = 8 * (32 // lpr) * 4
    return max(-(-max_inflight // per_block), 1) * 8 * (32 // lpr)


def mf_ordered_case(d, dtype):
    """1500 entries over 60 users and 80 items: rows repeat throughout, so the kernel's order protocol matters."""
    rng = np.random.default_rng([60, d, 0 if dtype == np.float32 else 1])
    nu, ni, n = 60, 80, 1500
    P = (rng.random((nu, d)) / 3).astype(dtype)
    Q = (rng.random((ni, d)) / 3).astype(dtype)
    u = rng.integers(0, nu, n).astype(np.int32)
    i = rng.integers(0, ni, n).astype(np.int32)
    r = (rng.integers(1, 9, n) / 2.0).astype(dtype)
    Bu, Bi = (rng.random(nu) / 5).astype(dtype), (rng.random(ni) / 5).astype(dtype)
    return dict(P=P, Q=Q, u=u, i=i, r=r, Bu=Bu, Bi=Bi)


# ---------------------------------------------------------------------------------------------------------------------
# SVD++ user-major epoch
SVDPP_DEGREES = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17, 18, 19, 33)    # W = 0, 1 and every residue mod kPrefetch


def svdpp_case(d, structure):
    """Users whose item counts W cycle through SVDPP_DEGREES, in a shuffled row order (users with W = 0 inside it),
    the last PAD columns of P, Q, Y zero, items no user rated.  'one_in_flight': items shared between users, one user
    at a time; 'disjoint': users share no item and max_users_in_flight = 7 lane groups take many users each."""
    rng = np.random.default_rng([70, d, ('one_in_flight', 'disjoint').index(structure)])
    nu = 120 if structure == 'one_in_flight' else 400
    deg = rng.permutation(np.resize(SVDPP_DEGREES, nu))
    rowptr = np.zeros(nu + 1, np.int64)
    rowptr[1:] = np.cumsum(deg)
    if structure == 'one_in_flight':
        ni = 300
        cols = np.concatenate([rng.choice(ni - 20, k, replace=False) for k in deg])
    else:
        ni = int(rowptr[-1]) + 50
        cols = rng.permutation(ni - 20)[:rowptr[-1]]
    vals = (rng.integers(1, 9, len(cols)) / 2.0).astype(np.float32)
    tabs = [rng.random((nu, d)) / 3, rng.random((ni, d)) / 3, rng.random((ni, d)), rng.random(nu), rng.random(ni)]
    tabs = [t.astype(np.float32) for t in tabs]
    for t in tabs[:3]:
        t[:, d - PAD:] = 0
    order = rng.permutation(nu)
    busy = np.nonzero(deg[order] > 0)[0][[0, -1]]       # users with items first and last, the empty ones between
    order = np.concatenate([order[busy[:1]], np.delete(order, busy), order[busy[1:]]]).astype(np.int32)
    return dict(tabs=tabs, rowptr=rowptr, cols=cols.astype(np.int32), vals=vals, order=order,
                in_flight=1 if structure == 'one_in_flight' else 7)


# ---------------------------------------------------------------------------------------------------------------------
# error measures
def zero_last_slice(tabs, d):
    """Copies of the tables with the last float4 of every row zeroed: what a kernel whose lane mask drops the last
    slice a lane group owns reads."""
    out = []
    for t in tabs:
        t = np.array(t, copy=True)
        if t.ndim == 2:
            t[:, d - 4:] = 0
        out.append(t)
    return out


def sum_ratio(got, ref, scale, unit=U32):
    """max |got - ref| / (unit * scale) over the elements, scale being the sum of the absolute values of the terms an
    element is made of (the fp32 summation error of a sum of n such terms is at most about n unit scale).  Elements
    with scale 0 must be exact."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    zero = scale == 0
    if np.any(err[zero] != 0):
        return math.inf
    return float((err[~zero] / (unit * scale[~zero])).max()) if (~zero).any() else 0.0


def table_ratio(got, ref, unit=U32, scale=None):
    """max |got - ref| in units of the table's rounding, unit * scale; scale defaults to max |ref|."""
    scale = np.abs(ref).max() if scale is None else scale
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / (unit * scale))


def loss_ratio(got, ref, unit=U32):
    return abs(float(got) - ref) / (unit * abs(ref))


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# Bounds, per launcher and output, in the units of the measure each output is judged by: sum_ratio for the SpMM
# outputs and K3's partial scores, table_ratio for tables and gradients (the staged step's deltas D against the
# magnitude of the staged rows they are differences of: (qin - lr regI qin) - qi rounds like qi, not like the delta),
# loss_ratio for losses.  Each fp32 bound is about 3 x the largest ratio observed over the launcher's cases on an H100
# 80GB HBM3 (700 W power limit), given beside it.  The float64 parity kernel is held to 1e-12 relative, as the
# golden-run tests hold it; it shows at most 9 units of 2^-53.
F64_REL = 1e-12 / U64
BOUNDS = {
    'spmm_balanced': {'Y': 15.0, 'acc': 15.0},                             # 5.4, 5.6
    'spmm_rowsplit': {'Y': 15.0, 'acc': 15.0},                             # 5.2, 5.2
    'spmm_scatter_rows': {'Y': 14.0, 'acc': 12.0},                         # 4.9, 4.2
    'spmm_rows': {'Y': 12.0, 'acc': 12.0},                                 # 4.2, 3.9
    'k3': {'gU': 3.5, 'gV': 3.0, 'y': 5.0, 'loss': 12.0},                  # 1.3, 1.0, 1.7, 4.3
    'bpr_staged': {'P': 4.5, 'D': 4.5, 'loss': 5.5},                       # 1.5, 1.5, 1.9
    'mf_batch': {'P': 2.5, 'Q': 2.5, 'Bu': 4.0, 'Bi': 4.0, 'loss': 2.0},   # 0.89, 0.90, 1.3, 1.4, 0.74
    'mf_ordered_f32': {'P': 27.0, 'Q': 25.0, 'Bu': 14.0, 'Bi': 8.5, 'loss': 1.2},  # 9.3, 8.6, 5.0, 2.9, 0.42
    'mf_ordered_f64': {'P': F64_REL, 'Q': F64_REL, 'Bu': F64_REL, 'Bi': F64_REL, 'loss': F64_REL},
    'svdpp_usermajor': {'P': 20.0, 'Q': 17.0, 'Y': 13.0, 'Bu': 19.0, 'Bi': 9.0, 'loss': 42.0},  # 7.0, 5.8, 4.6, 6.5, 3.0, 14
}
TEETH = 10.0           # the defective reference must lie at least this many bounds away


def judge(name, bounds, outputs):
    """outputs: {output: (observed, defect)} in the units of `bounds`.  Prints both over the bound and asserts that
    the kernel is inside every bound and the defective reference at least TEETH bounds outside it."""
    line = []
    for key, (obs, bad) in outputs.items():
        line.append('%s %.3g/%.3g' % (key, obs / bounds[key], bad / bounds[key]))
    print('\n%s observed/bound, defect/bound: %s' % (name, ', '.join(line)))
    for key, (obs, bad) in outputs.items():
        assert obs <= bounds[key], '%s: %s off by %.4g, bound %.4g' % (name, key, obs, bounds[key])
        assert bad >= TEETH * bounds[key], '%s: the %s bound cannot tell the defect (%.4g)' % (name, key, bad)
