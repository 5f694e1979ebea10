"""The float64 wave oracle of the user-major BPR epoch, and the table of cases it is applied to.

The epoch's launches run in waves (qrec_b200/csrc/um_waves.cuh).  Before a wave the item table is snapshotted; every
user of the wave runs its triples in order with P[u] updated after each one, reading item rows only from the snapshot;
the item-row deltas of the whole wave are summed into the table.  wave_oracle does exactly that in float64, with the
negatives the GPU drew.  What is left between the two is fp32 rounding and the summation order of the scatter-adds, far
below the difference that one user in a different wave would make.

A plain module, not collected: test_gpu_k1_schedule.py, test_gpu_k1_chain.py and test_gpu_k1_matrix.py apply the oracle
to the kernels, test_k1_wave_oracle_cpu.py checks the oracle itself and that every case below reaches the branch it is
named for."""
from collections import namedtuple

import numpy as np

CH = 32                         # um_waves.cuh: UM_CH


def row_lpr(nvec):
    """lane_shape.h: lanes per row of nvec float4s; the instantiation is FULL when d == 4 * row_lpr(d // 4)."""
    return 4 if nvec <= 4 else 8 if nvec <= 8 else 16 if nvec <= 16 else 32


def wave_chunks(n, num_items, d):
    """launch_usermajor's wave length in chunks of CH triples (um_wave_chunks)."""
    copy_bytes = 2 * num_items * d * 4
    copy_floor = 8 * copy_bytes // (24 * d + 12) if copy_bytes > (8 << 20) else 0
    return max(min(max(n // 64, copy_floor), 4 * num_items) // CH, 1)


def wave_oracle(P0, Q0, rowptr, i, j, launches, lr, reg_u, reg_i=None, shift=0):
    """float64 epoch: launches = [(ua, ub)], each a separate launch over users [ua, ub) with its own waves.  shift
    moves every wave boundary `shift` triples earlier.  reg_i defaults to reg_u.  The negatives j are data: whatever
    rejection sets they were drawn against (the positives' CSR or a superset of it) is the caller's business.

    One triple is bpr_step4_inplace in its folded form: pn = p + g (qi - qj); the item deltas g (1 - lr reg_i) pn
    - lr reg_i qi and -g (1 - lr reg_i) pn - lr reg_i qj are built from pn, not from the decayed row; then
    p = (1 - lr reg_u) pn."""
    from scipy import sparse
    P, Q = P0.astype(np.float64), Q0.astype(np.float64)
    a_u = lr * reg_u
    a_i = lr * (reg_u if reg_i is None else reg_i)
    loss = 0.0
    for ua, ub in launches:
        start = rowptr[ua:ub] - rowptr[ua]
        deg = np.diff(rowptr[ua:ub + 1])
        wave_of = (start + shift) // (wave_chunks(int(rowptr[ub] - rowptr[ua]), Q.shape[0], Q.shape[1]) * CH)
        users = np.arange(ua, ub)
        for w in np.unique(wave_of[deg > 0]):
            sel = (wave_of == w) & (deg > 0)
            uu, first, dg = users[sel], rowptr[ua:ub][sel], deg[sel]
            Qw = Q.copy()
            rows, deltas = [], []
            for k in range(int(dg.max())):
                on = dg > k
                u, t = uu[on], first[on] + k
                p, qi, qj = P[u], Qw[i[t]], Qw[j[t]]
                x = np.einsum('ij,ij->i', p, qi - qj)
                s = 1.0 / (1.0 + np.exp(-x))
                g = (lr * (1.0 - s))[:, None]
                loss += float(-np.log(s).sum())
                pn = p + g * (qi - qj)
                rows += [i[t], j[t]]
                deltas += [g * (1 - a_i) * pn - a_i * qi, -g * (1 - a_i) * pn - a_i * qj]
                P[u] = (1 - a_u) * pn
            r = np.concatenate(rows)
            S = sparse.csr_matrix((np.ones(len(r)), (r, np.arange(len(r)))), shape=(Q.shape[0], len(r)))
            Q += S @ np.concatenate(deltas)
    return P, Q, loss


def table_ratios(got_P, got_Q, P0, Q0, oracle):
    """max-abs distance of each table from the oracle's, as a fraction of the oracle's largest update of that table."""
    out = {}
    for got, ref, init, name in ((got_P, oracle[0], P0, 'P'), (got_Q, oracle[1], Q0, 'Q')):
        update = np.abs(ref - init).max()
        assert update > 0
        out[name] = float(np.abs(got.astype(np.float64) - ref).max() / update)
    return out


def check_against(got_P, got_Q, got_loss, P0, Q0, oracle, bound=1e-4, loss_bound=1e-5):
    """fp32 tables and an fp32 loss per lane against float64: at the d = 64, 5 000-item shape the rounding alone is
    about 3e-5 of the update on P.  Users run one wave early or late move the tables by far more
    (test_oracle_resolves_wave_membership).  bound is one number for both tables or a pair (P, Q).  Returns the ratios
    it prints."""
    bound_P, bound_Q = bound if isinstance(bound, tuple) else (bound, bound)
    errs = table_ratios(got_P, got_Q, P0, Q0, oracle)
    errs['loss'] = float(abs(got_loss - oracle[2]) / oracle[2])
    print('max-abs error over the largest update: P %.3g, Q %.3g; loss: relative error %.3g'
          % (errs['P'], errs['Q'], errs['loss']))
    assert errs['P'] <= bound_P and errs['Q'] <= bound_Q, errs
    assert errs['loss'] <= loss_bound, errs
    return errs


def pipeline_launches(rowptr, chunk):
    """The host pipeline's cut (qrec_bpr_epoch_usermajor_host): each launch takes the most whole users within `chunk`
    triples (and `chunk` users), at least one."""
    users = len(rowptr) - 1
    launches, ua = [], 0
    while ua < users:
        ub = int(np.searchsorted(rowptr, rowptr[ua] + chunk, side='right')) - 1
        ub = min(max(ub, ua + 1), users, ua + chunk)
        launches.append((ua, ub))
        ua = ub
    return launches


# ---------------------------------------------------------------------------------------------------------------------
# The cases of test_gpu_k1_matrix.py.
#
# degrees: ('tails',)        a shuffled cycle through 0 .. 2 LPR + 1, plus a block of users of degree exactly 1, G - 1,
#                            G, G + 1 (G = 2 and 4 triples in flight), LPR and LPR + 1: every tail of both loops
#          ('uniform', m)    uniform in 0 .. m
#          ('sparse', m)     one user in fifty has 1 .. m triples, the others none
#          ('long',)         users of 3 triples; two of 5 000 and 1 000 with an empty user between them, whose items
#                            repeat; one whose rated row holds every item
# entries: 'given' (negatives passed in), 'plain' / 'sig' (fused sampling), 'nojout' (plain, j_out absent),
#          'pipe' / 'pipe_sig' (HostPipeline with `chunk` triples per launch, without / with the rated signature)
# key:     (seed, epoch) of the Philox sampler
# tol, loss_tol: check_against's bounds (P, Q) and loss, each at most 3 x the ratio observed on an H100 80GB HBM3 (700 W
#          power limit).  Observed there, the same for every entry of a case: P 1.9e-5 (d = 4) .. 2.9e-5 (d = 100),
#          Q 7.4e-6 .. 9.7e-6 and loss 1.0e-7 .. 1.2e-7 over the widths.  That is nearly flat in d: the error is the
#          fp32 rounding of table entries near 0.3 accumulated over a user's triples, and in these cases the degrees,
#          and with them the largest update the error is measured against, grow with the lane-group size; the extra
#          terms of a wider dot product add little to it.  capped128 3.0e-5 / 1.3e-5,
#          large64 3.4e-5 / 7.2e-6, sparse32 3.0e-5 / 7.1e-6, pipe48 2.7e-5 / 7.8e-6, pipe128 2.9e-5 / 9.1e-6.
#          The long users are the exception: one lane group carries P[u] in fp32 through 5 000 sequential steps and
#          lane 0 sums the 5 000 losses in fp32 before the block adds them in double, so long16 shows 3.2e-5 / 2.6e-5
#          and 1.2e-6 on the loss, long64 4.2e-5 / 1.1e-5 and 3.8e-6.
Case = namedtuple('Case', 'name users items d degrees seed entries key chunk tol loss_tol')

BIG_KEY = (0x9e3779b97f4a7c15, 0x80000005)     # seed >> 32 != 0, epoch >= 2^31
SMALL_KEY = (0x5eed, 4)


TOL, LOSS_TOL = (5e-5, 2e-5), 3e-7             # (P, Q) and the loss


def _width(d):
    entries = ('given', 'plain') + (('sig',) if d in (16, 32, 64, 128) else ()) + (('nojout',) if d == 52 else ())
    return Case('w%d' % d, 8_000, 3_000, d, ('tails',), 100 + d, entries, BIG_KEY, 0, TOL, LOSS_TOL)


CASES = [_width(d) for d in (4, 12, 16, 20, 32, 48, 52, 64, 100, 128)] + [
    Case('long16', 300, 40, 16, ('long',), 16, ('given', 'plain', 'sig'), SMALL_KEY, 0, (9e-5, 7e-5), 3e-6),
    Case('long64', 300, 40, 64, ('long',), 64, ('given', 'plain', 'sig'), BIG_KEY, 0, (1.2e-4, 3e-5), 1e-5),
    Case('capped128', 8_000, 300, 128, ('uniform', 100), 7, ('given', 'plain', 'sig'), SMALL_KEY, 0, (5e-5, 3e-5), LOSS_TOL),
    Case('large64', 25_000, 40_000, 64, ('uniform', 120), 8, ('given', 'plain'), BIG_KEY, 0, (7e-5, 2e-5), LOSS_TOL),
    Case('sparse32', 200_000, 3_000, 32, ('sparse', 40), 9, ('given', 'plain', 'sig'), BIG_KEY, 0, TOL, LOSS_TOL),
    Case('pipe48', 8_000, 3_000, 48, ('tails',), 10, ('pipe', 'pipe_sig'), BIG_KEY, 20_000, TOL, LOSS_TOL),
    Case('pipe128', 8_000, 3_000, 128, ('tails',), 11, ('pipe', 'pipe_sig'), BIG_KEY, 40_000, TOL, LOSS_TOL),
]

LONG_USERS = {22: 5_000, 24: 1_000}            # test_k1_schedule_cpu.py: test_user_longer_than_a_wave's shape
SATURATED_USER, SATURATED_DEG = 40, 50


def case_degrees(case):
    rng = np.random.default_rng([case.seed, 0])
    kind = case.degrees[0]
    if kind == 'tails':
        lpr = row_lpr(case.d // 4)
        deg = rng.permutation(np.arange(case.users) % (2 * lpr + 2))
        edge = np.repeat([1, 2, 3, 4, 5, lpr, lpr + 1], 32)
        deg[case.users // 2:case.users // 2 + len(edge)] = edge
    elif kind == 'uniform':
        deg = rng.integers(0, case.degrees[1] + 1, case.users)
    elif kind == 'sparse':
        deg = np.zeros(case.users, np.int64)
        deg[rng.choice(case.users, case.users // 50, replace=False)] = rng.integers(1, case.degrees[1] + 1, case.users // 50)
    else:
        deg = np.full(case.users, 3, np.int64)
        for u, k in LONG_USERS.items():
            deg[u] = k
        deg[23] = 0
        deg[SATURATED_USER] = SATURATED_DEG
    return deg.astype(np.int64)


def case_rowptr(case):
    rowptr = np.zeros(case.users + 1, np.int64)
    rowptr[1:] = np.cumsum(case_degrees(case))
    return rowptr


def case_launches(case, rowptr):
    return pipeline_launches(rowptr, case.chunk) if case.chunk else [(0, case.users)]


THRESHOLD = 3.0                                 # ratings 1 .. 5; a positive is a rating of 3 or more


def case_data(case, E):
    """The epoch's triples and its rejection sets, which are a strict superset of the positives: about a third of
    every user's ratings are under the threshold.  E is qrec_b200.engine (RatedCSR is host code)."""
    rng = np.random.default_rng([case.seed, 1])
    rowptr = case_rowptr(case)
    deg = np.diff(rowptr)
    uu, ii, is_pos = [], [], []
    direct = {}                                                   # 'long': users whose triples repeat items
    for u in np.nonzero(deg)[0]:
        k = int(deg[u])
        if case.degrees[0] == 'long' and k > 3:
            # the long users rate 30 of the 40 items (20 of them positives), so most draws are rejected at least
            # once; the saturated user rates them all, its negatives are first draws and may equal i
            rated = rng.permutation(case.items)[:case.items if u == SATURATED_USER else 30]
            pos = np.zeros(len(rated), bool)
            pos[:2 * len(rated) // 3] = True
            direct[u] = rng.choice(rated[pos], k, replace=True)
        else:
            rated = rng.choice(case.items, k + (k + 1) // 2, replace=False)
            pos = rng.permutation(len(rated)) < k
        uu.append(np.full(len(rated), u))
        ii.append(rated)
        is_pos.append(pos)
    uu, ii, is_pos = np.concatenate(uu), np.concatenate(ii), np.concatenate(is_pos)
    ratings = np.where(is_pos, rng.integers(3, 6, len(uu)), rng.integers(1, 3, len(uu))).astype(np.float64)
    csr = E.RatedCSR(case.users, case.items, uu, ii, ratings=ratings, positive_threshold=THRESHOLD)
    if direct:
        i = np.concatenate([direct[u] if u in direct else csr.pos_cols[csr.pos_rowptr[u]:csr.pos_rowptr[u + 1]]
                            for u in range(case.users)]).astype(np.int32)
    else:
        assert np.array_equal(csr.pos_rowptr, rowptr)
        i = csr.pos_cols
    assert len(i) == rowptr[-1] and csr.sorted_rowptr[-1] > csr.pos_rowptr[-1]
    u = np.repeat(np.arange(case.users), deg).astype(np.int32)
    return dict(rowptr=rowptr, u=u, i=np.ascontiguousarray(i), rated_rowptr=csr.sorted_rowptr, rated_cols=csr.sorted_cols)


def case_tables(case):
    rng = np.random.default_rng([case.seed, 2])
    return (rng.random((case.users, case.d)) / 3).astype(np.float32), (rng.random((case.items, case.d)) / 3).astype(np.float32)
