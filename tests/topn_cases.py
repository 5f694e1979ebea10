"""Exact-score cases and references for the two K8 top-N kernels (qrec_b200/csrc/topn_kernels.cu, the fp32 SIMT
kernel, and qrec_b200/csrc/topn_tc.cu, the wgmma 3xTF32 kernel) and for `evaluate.batched_top_n`, the `-eval gpu`
ranking that every model with `device_tables()` goes through.

Every table entry is an integer with |x| <= 8 and d <= 256, so every product and partial sum is an integer of magnitude
at most 2^14: any summation order, fmaf or TF32 gives the float64 score (the TF32 split of an entry is hi = x, lo = 0).
The kernels' ids and scores can therefore be compared with the references bit for bit, ties included.

Two references:
  kernel_reference -- the contract of engine.score_topn: rated items score `rated_value`, then (score descending,
                      item id ascending), +0.0 and -0.0 one score;
  heap_reference   -- the contract of `-eval gpu`: util.qmath.find_k_largest (the reference's min-heap of
                      (score, id) with a strict `>` replace) on the same row, rated items scored 0.

The cases cover both kernels' constants (below): widths on both sides of every k-chunk and k-block, row counts around
a CTA and a 32-row quarter, item counts around a tile and a half-tile, N from 1 to 101 and N = n_items, score rows
that compact every tile, tie at every compaction and at the cut, rated rows that are empty, longer than the rated
signature, complete and straddling the cut, and zero user rows whose products are all -0.0.

`DEFECTS` are plausible wrong references; test_topn_cases_cpu.py proves that each family of cases tells the ones it
targets apart from the true reference.  A plain module, not collected: test_gpu_topn_matrix.py runs the kernels on
the cases."""
import numpy as np

# ---------------------------------------------------------------------------------------------------------------------
# kernel constants
SIMT_VM, SIMT_VN, SIMT_VK, SIMT_CAP = 128, 128, 16, 256     # users per CTA, items per tile, k-chunk, list slots
TC_TM, TC_TN, TC_HALF = 128, 128, 64                         # users per CTA, items per tile, columns per half-list
TC_CAP, TC_TRIG, TC_SORTN = 320, 96, 256                     # list slots, compaction trigger above N, merge sort keys
TC_SIGBITS, TC_QUARTER = 512, 32                             # rated-signature bits per row, rows per selecting warp
NMAX = 101

SIMT_D = (1, 3, 4, 15, 16, 17, 31, 32, 33, 64, 100, 128, 129, 256)
TC_D = (4, 8, 28, 32, 36, 52, 60, 64)
ROWS = (1, 31, 32, 33, 127, 128, 129, 257)
NS = (1, 2, 10, 32, 33, 100, 101)

SENTINEL_ID = -7
SENTINEL_BITS = 0x7FC0DEAD        # a NaN no kernel writes


def tc_ok(d):
    """the tensor-core kernel takes d <= 64, a multiple of 4"""
    return d <= 64 and d % 4 == 0


class Case:
    def __init__(self, name, family, U, V, users, rowptr, cols, rated_value, N):
        self.name, self.family = name, family
        self.U, self.V = U, V
        self.users, self.rowptr, self.cols = users, rowptr, cols
        self.rated_value, self.N = float(rated_value), int(N)

    d = property(lambda self: self.U.shape[1])
    n_items = property(lambda self: self.V.shape[0])
    n_rows = property(lambda self: len(self.users))
    kernels = property(lambda self: ('simt', 'tc') if tc_ok(self.d) else ('simt',))

    def __repr__(self):
        return self.name


# ---------------------------------------------------------------------------------------------------------------------
# keys: (ord(score) << 32) | (0xffffffff - id), the kernels' 64-bit candidate keys; descending keys are
# (score descending, id ascending)
def ord_of(s32):
    u = np.asarray(s32, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)


def make_keys(s32, ids):
    return (ord_of(s32) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - ids.astype(np.uint64))


def scores64(U, V, users):
    """float64 scores [len(users), n_items], exact; +0.0 for every zero"""
    return U.astype(np.float64)[users] @ V.astype(np.float64).T + 0.0


def rated_mask(rowptr, cols, users, n_items):
    m = np.zeros((len(users), n_items), bool)
    for r, u in enumerate(users):
        m[r, cols[rowptr[u]:rowptr[u + 1]]] = True
    return m


# ---------------------------------------------------------------------------------------------------------------------
# references
def _signed_zero_scores(U, V, users, S):
    """S with the IEEE sign of a zero sum whose first term is a product (an accumulator that starts from the first
    product rather than +0): -0.0 where every product is -0.0"""
    P = U.astype(np.float64)[users][:, None, :] * V.astype(np.float64)[None, :, :]
    neg = np.all((P == 0) & np.signbit(P), axis=2)
    return np.where(neg & (S == 0), -0.0, S)


def topn(U, V, users, rowptr, cols, N, rated_value, defect=None):
    """(ids int64 [n, N], scores float32 [n, N]) by (score descending, id ascending) -- the kernel contract -- or by one
    of DEFECTS.  A defect that leaves fewer than N candidates pads with id -1 and a NaN score."""
    users = np.asarray(users)
    uniq, inv = np.unique(users, return_inverse=True)
    n_items, d = V.shape[0], V.shape[1]
    if defect == 'last_column':
        U, V = U.copy(), V.copy()
        U[:, d - 1] = 0
        V[:, d - 1] = 0
    S = scores64(U, V, uniq)
    if defect == 'neg_zero':
        S = _signed_zero_scores(U, V, uniq, S)
    s32 = S.astype(np.float32)
    rated = rated_mask(rowptr, cols, uniq, n_items)
    s32[rated] = np.float32(rated_value)
    if defect != 'neg_zero':
        s32 = s32 + np.float32(0.0)                   # one zero
    ids = np.arange(n_items, dtype=np.int64)
    out_i = np.full((len(uniq), N), -1, np.int64)
    out_s = np.full((len(uniq), N), np.nan, np.float32)
    for r in range(len(uniq)):
        keep = np.ones(n_items, bool)
        if defect == 'rated_removed':
            keep &= ~rated[r]
        if defect == 'last_tile':
            keep &= ids < (n_items - 1) // SIMT_VN * SIMT_VN
        s, k = s32[r][keep], ids[keep]
        if defect == 'ties_desc':
            order = np.lexsort((-k, -s.astype(np.float64)))
        else:
            key = make_keys(s, k)
            order = np.argsort(key)[::-1]
        order = order[:N]
        out_i[r, :len(order)] = k[order]
        out_s[r, :len(order)] = s[order]
    return out_i[inv], out_s[inv]


def heap_topn(U, V, users, rowptr, cols, N, rated_value=0.0):
    """util.qmath.find_k_largest on every row (rated items scored `rated_value`): (ids int64, scores float32)"""
    from qrec_b200.util.qmath import find_k_largest
    users = np.asarray(users)
    uniq, inv = np.unique(users, return_inverse=True)
    n_items = V.shape[0]
    N = min(N, n_items)
    S = scores64(U, V, uniq)
    S[rated_mask(rowptr, cols, uniq, n_items)] = rated_value
    out_i = np.empty((len(uniq), N), np.int64)
    out_s = np.empty((len(uniq), N), np.float32)
    for r in range(len(uniq)):
        k, v = find_k_largest(N, S[r])
        out_i[r], out_s[r] = k, v
    return out_i[inv], out_s[inv]


def kernel_reference(case, rated_value=None, defect=None):
    rv = case.rated_value if rated_value is None else rated_value
    return topn(case.U, case.V, case.users, case.rowptr, case.cols, case.N, rv, defect)


def driver_n(case):
    """N of the case for evaluate.batched_top_n, which takes N <= 100 (the recommender's clamp)"""
    return min(case.N, 100)


def heap_reference(case, rated_value=0.0):
    return heap_topn(case.U, case.V, case.users, case.rowptr, case.cols, driver_n(case), rated_value)


# defect -> what it restates wrongly
DEFECTS = {
    'ties_desc': 'ties broken by descending item id',
    'kernel_for_heap': 'ties by ascending id where the reference heap is required',
    'rated_removed': 'rated items removed instead of scored',
    'last_tile': 'the last item tile dropped',
    'last_column': 'the last column of d dropped',
    'neg_zero': '-0.0 ordered below +0.0',
}
# family -> the defects each of its cases is built to expose (at least one case of the family must)
FAMILY_TARGETS = {
    'width': ('last_column', 'ties_desc', 'rated_removed', 'last_tile'),
    'rows': ('ties_desc', 'rated_removed', 'last_column', 'kernel_for_heap'),
    'items': ('last_tile', 'ties_desc', 'rated_removed', 'last_column'),
    'ties': ('ties_desc', 'kernel_for_heap', 'last_tile', 'last_column'),
    'rated': ('rated_removed', 'kernel_for_heap', 'ties_desc'),
    'zero': ('neg_zero', 'kernel_for_heap', 'ties_desc'),
    'driver': ('kernel_for_heap', 'ties_desc', 'rated_removed'),
}


def defect_output(case, defect):
    """what a defective kernel would return on the case, and what the true contract returns"""
    if defect == 'kernel_for_heap':
        return topn(case.U, case.V, case.users, case.rowptr, case.cols, driver_n(case), 0.0), heap_reference(case)
    return kernel_reference(case, defect=defect), kernel_reference(case)


def same_output(a, b):
    """ids equal and scores equal bit for bit"""
    (ia, sa), (ib, sb) = a, b
    return ia.shape == ib.shape and np.array_equal(ia, ib) and np.array_equal(sa.view(np.uint32), sb.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# builders
def _split(t, d, rng):
    """integer rows [len(t), d], entries in [-8, 8], row k summing to t[k] (|t| <= 8 d), the sum spread at random"""
    t = np.asarray(t, np.int64)
    base = np.floor_divide(t, d)
    X = np.repeat(base[:, None], d, axis=1)
    rem = t - base * d
    X[np.arange(d)[None, :] >= d - rem[:, None]] += 1       # the remainder on the last columns: they carry weight
    for _ in range(3 if d > 1 else 0):                        # random transfers between column pairs keep the sums
        perm = rng.permutation(d)
        a, b = perm[: d // 2], perm[d // 2: 2 * (d // 2)]
        xa, xb = X[:, a], X[:, b]
        lo = np.maximum(xa - 8, -8 - xb)
        hi = np.minimum(xa + 8, 8 - xb)
        delta = lo + np.floor(rng.random(lo.shape) * (hi - lo + 1)).astype(np.int64)
        X[:, a], X[:, b] = xa - delta, xb + delta
    assert np.all(np.abs(X) <= 8) and np.array_equal(X.sum(axis=1), t)
    return X


def _levels(structure, n_items, d, rng):
    R = 8 * d
    i = np.arange(n_items)
    if structure == 'asc':                                    # ascending in id: the row compacts every tile
        return -R + (2 * R * i) // max(n_items - 1, 1)
    if structure == 'desc':
        return R - (2 * R * i) // max(n_items - 1, 1)
    if structure == 'equal':
        return np.full(n_items, R // 2)
    if structure == 'levels4':                                # four values: ties meet every compaction and the cut
        return np.array([-R // 2, 0, R // 4 + 1, R])[rng.integers(0, 4, n_items)]
    if structure == 'levels3':
        return np.array([-1, 0, 1])[rng.integers(0, 3, n_items)]
    raise ValueError(structure)


def _items(structure, n_items, d, rng):
    if structure == 'zero':                                   # every third row all negative, the rest mixed in sign
        V = rng.integers(-8, 9, (n_items, d))
        V[:, 0] = np.abs(V[:, 0])
        neg = np.arange(n_items) % 3 == 0
        V[neg] = -rng.integers(1, 9, (int(neg.sum()), d))
        return V
    return _split(_levels(structure, n_items, d, rng), d, rng)


USER_KINDS = ('one', 'neg', 'rand', 'one', 'rand', 'neg')


def _user_rows(kinds, d, rng):
    U = np.zeros((len(kinds), d), np.int64)
    for r, k in enumerate(kinds):
        if k == 'one':
            U[r] = 1
        elif k == 'neg':
            U[r] = -1
        elif k == 'rand':
            U[r] = rng.integers(-8, 9, d)
        elif k == 'two':
            U[r] = 2
        else:
            assert k == 'zero'
    return U


RATED_KINDS = ('none', 'cut', 'rand', 'long', 'all', 'cut')


def _rated_rows(kinds, U, V, N, rng):
    n_items = V.shape[0]
    rows = []
    for u, kind in enumerate(kinds):
        if kind == 'none':
            r = np.zeros(0, np.int64)
        elif kind == 'all':
            r = np.arange(n_items)
        elif kind == 'long':                                   # more than the signature's 512 bits when there are items
            r = np.sort(rng.choice(n_items, min(n_items, max(TC_SIGBITS + 40, n_items * 7 // 8)), replace=False))
        elif kind == 'rand':
            r = np.sort(rng.choice(n_items, max(1, n_items // 10), replace=False))
        else:                                                  # above, at and below the cut of the unrated ranking
            assert kind == 'cut'
            s = scores64(U, V, [u])[0]
            order = np.lexsort((np.arange(n_items), -s))
            pos = np.array([0, N // 2, N - 1, N, N + 1, 2 * N + 3, n_items - 1])
            r = np.unique(order[pos[pos < n_items]])
        rows.append(np.asarray(r, np.int64))
    rowptr = np.zeros(len(rows) + 1, np.int64)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    cols = np.concatenate(rows + [np.zeros(0, np.int64)]).astype(np.int32)
    return rowptr, cols


def _user_list(nu, n_rows, rng):
    """n_rows rows of user ids: every user once (while rows last), then repeats, in random order"""
    base = rng.permutation(nu)
    users = np.concatenate([base, rng.integers(0, nu, max(0, n_rows - nu))])[:n_rows]
    return rng.permutation(users).astype(np.int32)


RATED_VALUES = ('zero', 'above', 'below', 'between')


def _rated_value(which, d):
    top = 64.0 * d
    return {'zero': 0.0, 'negzero': -0.0, 'above': top + 1.0, 'below': -top - 1.0, 'between': 2.5}[which]


def build(name, family, d, n_items, n_rows, N, structure, seed, user_kinds=USER_KINDS, rated_kinds=RATED_KINDS,
          rated_value='zero'):
    assert 1 <= N <= min(NMAX, n_items) and d <= 256
    rng = np.random.default_rng(seed)
    V = _items(structure, n_items, d, rng)
    U = _user_rows(user_kinds, d, rng)
    rk = [rated_kinds[k % len(rated_kinds)] for k in range(len(user_kinds))]
    rowptr, cols = _rated_rows(rk, U, V, N, rng)
    users = _user_list(len(user_kinds), n_rows, rng)
    return Case(name, family, U.astype(np.float32), V.astype(np.float32), users, rowptr, cols,
                _rated_value(rated_value, d), N)


def _cycle(seq, k):
    return seq[k % len(seq)]


def _cases():
    out = []
    structures = ('asc', 'levels4', 'desc', 'equal', 'levels3')
    # every width of both kernels: k-chunk / k-block tails and multiples
    for k, d in enumerate(sorted(set(SIMT_D) | set(TC_D))):
        ni = _cycle((200, 257, 300, 129, 385), k)
        N = min(_cycle(NS, k), ni)
        out.append(build('width_d%d_i%d_N%d' % (d, ni, N), 'width', d, ni, _cycle(ROWS, k), N,
                         _cycle(structures, k), 100 + k, rated_value=_cycle(RATED_VALUES, k)))
    # every row count: partial CTAs and 32-row quarters, repeated users
    for k, nr in enumerate(ROWS):
        d = _cycle(TC_D, k)
        out.append(build('rows_r%d_d%d' % (nr, d), 'rows', d, _cycle((130, 300), k), nr, _cycle((10, 33, 100), k),
                         _cycle(('levels4', 'asc', 'levels3'), k), 200 + k))
    # item counts around a tile and a half-tile, N up to n_items
    items_n = ((1, 1), (2, 2), (2, 1), (10, 10), (33, 32), (33, 33), (63, 10), (64, 64), (65, 33), (100, 100),
               (101, 101), (127, 100), (128, 101), (129, 2), (191, 101), (192, 32), (193, 1), (255, 100), (256, 10),
               (257, 101), (300, 33))
    for k, (ni, N) in enumerate(items_n):
        d = _cycle((4, 32, 36, 64, 17, 100, 8, 3, 60), k)
        out.append(build('items_i%d_N%d_d%d' % (ni, N, d), 'items', d, ni, _cycle(ROWS, k + 3), N,
                         _cycle(structures, k), 300 + k, rated_value=_cycle(RATED_VALUES, k + 1)))
    # ties at every compaction and at the cut
    for k, (structure, ni, N, d) in enumerate((
            ('equal', 700, 100, 4), ('equal', 300, 101, 32), ('levels4', 700, 10, 64), ('levels4', 700, 101, 36),
            ('levels3', 700, 33, 8), ('levels3', 700, 100, 64), ('levels3', 260, 1, 3), ('asc', 700, 100, 1),
            ('asc', 700, 1, 32), ('levels4', 500, 32, 128), ('equal', 640, 2, 52), ('levels3', 900, 101, 16))):
        out.append(build('ties_%s_i%d_N%d_d%d' % (structure, ni, N, d), 'ties', d, ni, _cycle(ROWS, k + 5), N,
                         structure, 400 + k, user_kinds=('one', 'two', 'neg', 'rand', 'one', 'neg'),
                         rated_kinds=('none', 'cut', 'none', 'rand', 'none', 'cut'),
                         rated_value=_cycle(RATED_VALUES, k)))
    # rated rows: empty, longer than the signature, complete, across the cut; every rated value
    for k, (rv, d, ni, N) in enumerate((('zero', 8, 700, 100), ('above', 64, 700, 101), ('below', 16, 700, 10),
                                        ('between', 32, 700, 33), ('zero', 129, 600, 100), ('between', 4, 600, 101),
                                        ('above', 33, 300, 32), ('below', 60, 300, 100))):
        out.append(build('rated_%s_d%d_i%d_N%d' % (rv, d, ni, N), 'rated', d, ni, _cycle(ROWS, k + 1), N,
                         _cycle(structures, k), 500 + k, user_kinds=('rand', 'one', 'neg', 'rand', 'one', 'two'),
                         rated_kinds=('long', 'all', 'cut', 'none', 'cut', 'long'), rated_value=rv))
    # zero user rows against item rows whose products are all -0.0 or mixed in sign
    # (and a rated value of -0.0, which ties with every +0.0 score)
    for k, (d, ni, N, rv) in enumerate(((4, 200, 10, 'zero'), (32, 200, 100, 'zero'), (64, 130, 33, 'zero'),
                                        (1, 200, 10, 'zero'), (33, 300, 101, 'zero'), (8, 64, 64, 'zero'),
                                        (4, 200, 10, 'negzero'), (33, 300, 100, 'negzero'))):
        out.append(build('zero_d%d_i%d_N%d%s' % (d, ni, N, '_rated_negzero' if rv == 'negzero' else ''), 'zero', d, ni,
                         _cycle(ROWS, k + 2), N, 'zero', 600 + k, user_kinds=('zero', 'one', 'zero', 'rand'),
                         rated_kinds=('none', 'rand', 'cut', 'none'), rated_value=rv))
    # the tie pattern of the hand-made kernel test: rated zeros above an all-negative row, a tie block across the cut
    for d in (4, 32, 64, 17):
        U = np.zeros((3, d), np.float32)
        U[:, :4] = 1.0
        V = np.zeros((400, d), np.float32)
        V[:, :4] = -2.0                                       # every raw score -8
        V[100:110, :4] = -1.0                                 # a block of ten at -4
        rowptr = np.array([0, 5, 5, 9], np.int64)
        cols = np.array([3, 50, 150, 250, 399, 0, 1, 2, 398], np.int32)
        out.append(Case('driver_d%d' % d, 'driver', U, V, np.arange(3, dtype=np.int32), rowptr, cols, 0.0, 12))
    return out


CASES = _cases()


# ---------------------------------------------------------------------------------------------------------------------
# what the kernels do with a case: list lengths, compactions and branches, simulated from the constants above
def _row_keys(case, u):
    """(raw keys, keys with rated items at rated_value, rated mask) of user u"""
    s = scores64(case.U, case.V, [u])[0].astype(np.float32) + np.float32(0.0)
    ids = np.arange(case.n_items)
    rated = rated_mask(case.rowptr, case.cols, [u], case.n_items)[0]
    eff = s.copy()
    eff[rated] = np.float32(case.rated_value)
    return make_keys(s, ids), make_keys(eff + np.float32(0.0), ids), rated


def _sig_bits(cols):
    h = ((cols.astype(np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) >> np.uint64(23)
    return np.unique(h)


def simt_paths(case):
    """branches of score_topn_kernel the case reaches; the simulated result is checked against kernel_reference"""
    paths = set()
    N, ni, d = case.N, case.n_items, case.d
    paths.add('k_tail' if d % SIMT_VK else 'k_full')
    if d > SIMT_VK:
        paths.add('k_chunks')
    if case.n_rows % SIMT_VM:
        paths.add('cta_tail')
    if ni % SIMT_VN:
        paths.add('tile_tail')
    for u in np.unique(case.users):
        raw, eff, rated = _row_keys(case, u)
        lst, thr = np.zeros(0, np.uint64), np.uint64(0)
        for c0 in range(0, ni, SIMT_VN):
            if len(lst) > SIMT_CAP - SIMT_VN:
                srt = np.sort(lst)[::-1]
                if (srt[N - 1] >> np.uint64(32)) == (srt[N] >> np.uint64(32)):
                    paths.add('compact_tie_at_cut')            # equal scores on both sides of the cut
                lst, thr = srt[:N], srt[N - 1]
                paths.add('compact')
            sl = slice(c0, min(ni, c0 + SIMT_VN))
            passed = eff[sl] > thr
            if np.any(passed & ~(raw[sl] > thr)):
                paths.add('rated_rescued')                     # only the rated value lets it pass
            if np.any(~passed & (raw[sl] > thr) & rated[sl]):
                paths.add('rated_demoted')
            lst = np.concatenate([lst, eff[sl][passed]])
            assert len(lst) <= SIMT_CAP
        assert len(lst) >= N
        top = np.sort(lst)[::-1][:N]
        ref_i, _ = kernel_reference(case)
        row = int(np.nonzero(case.users == u)[0][0])
        assert np.array_equal(np.uint64(0xFFFFFFFF) - (top & np.uint64(0xFFFFFFFF)), ref_i[row].astype(np.uint64))
    return paths


def tc_paths(case):
    """branches of score_topn_tc_kernel<KB> the case reaches; the simulated result is checked against kernel_reference"""
    assert tc_ok(case.d)
    paths = set()
    N, ni, d = case.N, case.n_items, case.d
    paths.add('kb1' if d <= 32 else 'kb2')
    if d % 32:
        paths.add('k_pad')
    tail = case.n_rows % TC_TM
    if tail:
        paths.add('cta_tail')
    if case.n_rows % TC_QUARTER:
        paths.add('quarter_tail')
    if tail and tail <= TC_TM - TC_QUARTER:
        paths.add('empty_quarter')
    n_tiles = (ni + TC_TN - 1) // TC_TN
    rkh = ord_of(np.float32(case.rated_value)) << np.uint64(32)
    hi = lambda k: k >> np.uint64(32)                          # noqa: E731
    ref_i, _ = kernel_reference(case)
    for u in np.unique(case.users):
        raw, eff, rated = _row_keys(case, u)
        rc = case.cols[case.rowptr[u]:case.rowptr[u + 1]]
        sig = _sig_bits(rc)
        if len(sig) == TC_SIGBITS:
            paths.add('sig_saturated')
        sig_set = set(sig.tolist())
        lists = [np.zeros(0, np.uint64), np.zeros(0, np.uint64)]
        thrs = [np.uint64(0), np.uint64(0)]

        def compact(h, final):
            lst = lists[h]
            cut = np.sort(lst)[::-1][N - 1]
            above = int(np.sum(hi(lst) > hi(cut)))
            equal = int(np.sum(hi(lst) == hi(cut)))
            if equal > N - above:
                paths.add('tie_search_final' if final else 'tie_search')
            paths.add('compact_final' if final else 'compact')
            lists[h] = lst[lst >= cut]
            assert len(lists[h]) == N
            thrs[h] = cut

        for t in range(n_tiles):
            for h in (0, 1):
                if len(lists[h]) > N + TC_TRIG:
                    compact(h, False)
                c0 = t * TC_TN + h * TC_HALF
                valid = ni - c0
                if valid <= 0:
                    paths.add('empty_half')
                    continue
                if valid < TC_HALF:
                    paths.add('half_tail')
                    if valid % 16:
                        paths.add('group_tail')
                thr = thrs[h]
                open_row = thr == 0 or hi(thr) <= hi(rkh)
                if thr != 0 and open_row:
                    paths.add('open_row')
                sl = slice(c0, c0 + min(valid, TC_HALF))
                # the float pre-filter: score >= the cut-off's score (the scores here carry one zero)
                pre = np.ones(sl.stop - sl.start, bool) if open_row else hi(raw[sl]) >= hi(thr)
                cand = pre & ((raw[sl] > thr) | ((rkh | (raw[sl] & np.uint64(0xFFFFFFFF))) > thr))
                items = np.arange(sl.start, sl.stop)
                hits = np.array([(((int(c) * 0x9E3779B1) & 0xFFFFFFFF) >> 23) in sig_set for c in items[cand]], bool)
                if np.any(hits & ~rated[sl][cand]):
                    paths.add('sig_false_hit')
                passed = eff[sl] > thr
                assert np.all(cand | ~passed)
                if np.any(passed & ~(raw[sl] > thr)):
                    paths.add('rated_rescued')
                lists[h] = np.concatenate([lists[h], eff[sl][passed]])
                assert len(lists[h]) <= TC_CAP
        for h in (0, 1):
            if len(lists[h]) > N:
                compact(h, True)
        if len(lists[1]) == 0:
            paths.add('second_list_empty')
        merged = np.concatenate(lists)
        assert len(merged) <= TC_SORTN and len(merged) >= N
        top = np.sort(merged)[::-1][:N]
        row = int(np.nonzero(case.users == u)[0][0])
        assert np.array_equal(np.uint64(0xFFFFFFFF) - (top & np.uint64(0xFFFFFFFF)), ref_i[row].astype(np.uint64))
    return paths


# ---------------------------------------------------------------------------------------------------------------------
# exactness: how the kernels would compute the scores
def fma_scores_f32(U, V, users):
    """score_topn_kernel's sums: fp32 accumulators from +0, k ascending, one fmaf per k; returns (scores, max |partial|)"""
    A = U.astype(np.float64)[users]
    B = V.astype(np.float64)
    acc = np.zeros((A.shape[0], B.shape[0]), np.float32)
    peak = 0.0
    for k in range(A.shape[1]):
        exact = acc.astype(np.float64) + A[:, k:k + 1] * B[None, :, k]   # fmaf: one rounding of product + sum
        peak = max(peak, float(np.abs(exact).max()))
        acc = exact.astype(np.float32)
    return acc, peak


def tf32_rna(x):
    """cvt.rna.tf32.f32: round to the nearest TF32 (10 mantissa bits), ties away from zero"""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return r.view(np.float32)


def tf32_split(x):
    x = np.asarray(x, np.float32)
    hi = tf32_rna(x)
    return hi, tf32_rna(x - hi)


# ---------------------------------------------------------------------------------------------------------------------
# end to end: a recommender over integer tables, ranked by Recommender.evalRanking with `-topN 5,10`
def tie_model(d, out_dir, device, gpu_eval):
    """A Recommender whose scores are small integers (ties inside every top-10 and across its cut; rated items score
    0 and tie with the zero scores), run through execute() with or without `engine=-eval gpu`.  Returns the model."""
    import contextlib
    import io
    from qrec_b200.base.recommender import Recommender
    from qrec_b200.util.config import ModelConf
    nu, ni = 40, 60
    rng = np.random.default_rng(d)
    train, rated = [], [set() for _ in range(nu)]
    for i in range(ni):                                   # every item rated by someone, some users rate several
        for u in {i % nu, (7 * i) % 13}:
            train.append(['u%d' % u, 'i%d' % i, 1.0])
            rated[u].add(i)
    test = []
    for u in range(nu):
        test += [['u%d' % u, 'i%d' % i, 1.0] for i in [i for i in rng.permutation(ni) if i not in rated[u]][:3]]
    lines = ['ratings=./ratings.txt', 'ratings.setup=-columns 0 1 2', 'model.name=TieRank',
             'evaluation.setup=-ap 0.2', 'item.ranking=on -topN 5,10', 'output.setup=on -dir %s/' % out_dir]
    if gpu_eval:
        lines.append('engine=-eval gpu')

    class TieRank(Recommender):
        def initModel(self):
            g = np.random.default_rng(1000 + d)
            self.P = (g.integers(1, 3, (self.num_users, d)) * g.choice([-1, 1], (self.num_users, d))).astype(np.float64)
            self.Q = g.integers(-2, 3, (self.num_items, d)).astype(np.float64)
            self.Q[:, 0] = g.choice([-2, -1, 1, 2], self.num_items)     # no row of zero products: no -0.0 on the host

        def predictForRanking(self, u):
            return self.Q.dot(self.P[self.data.user[u]])

        def device_tables(self):
            import torch
            return tuple(torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(device) for X in (self.P, self.Q))

    model = TieRank(ModelConf.from_string('\n'.join(lines)), train, test)
    with contextlib.redirect_stdout(io.StringIO()):
        model.execute()
    return model
