"""The engine wrappers' argument checks on CPU tensors, without a GPU.

A checking wrapper raises QRecError in three steps: shapes, lengths and dtypes; then that every tensor is a contiguous
CUDA tensor; then the contents, which need reductions on the device.  So on CPU tensors every shape, length or dtype
fault raises its own message, and a call whose shapes are valid stops at the device check, whatever its contents.

The *_cases builders return (call, message, contents) triples on the given device; tests/test_gpu_engine_checks.py
runs their contents cases on CUDA tensors, where each must raise its own message."""
import numpy as np
import pytest

CUDA = 'must be a CUDA tensor'


def check_cases(cases, on_device):
    """Every call raises QRecError matching its message; on CPU tensors (not on_device) a contents case stops at the
    device check instead.  On the device only the contents cases run."""
    from qrec_b200 import engine as E
    for k, (call, message, contents) in enumerate(cases):
        if on_device and not contents:
            continue
        with pytest.raises(E.QRecError, match=message if on_device or not contents else CUDA):
            call()
            pytest.fail('case %d (%s) did not raise' % (k, message))


def _csr(rows):
    rowptr = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    return rowptr, np.array([c for r in rows for c in r], np.int32)


def _t(torch, device, a, dtype=None):
    return torch.as_tensor(a, dtype=dtype).to(device)


def _exposure_problem(torch, device):
    """X [5, 3] against Z [4, 3] with a CSR of X's rows into Z's."""
    rowptr, cols = _csr([[0, 2], [1], [], [3, 0, 1], [2]])
    return (torch.rand(5, 3, device=device), torch.rand(4, 3, device=device), _t(torch, device, rowptr),
            _t(torch, device, cols), torch.arange(5, dtype=torch.int32, device=device))


def expomf_cases(torch, device):
    from qrec_b200 import engine as E
    X, Z, rp, cl, order = _exposure_problem(torch, device)
    mz, mx = torch.full((4,), 0.1, device=device), torch.full((5,), 0.1, device=device)

    def half(X=X, Z=Z, rowptr=rp, cols=cl, mu=mz, by_row=False, order=order, **kw):
        return lambda: E.expomf_half_epoch(X, Z, rowptr, cols, mu, by_row, 1e-5, 1.0, order, **kw)

    return [
        (half(X=X.double()), 'expomf_half_epoch: X must be float32, got torch.float64', False),
        (half(Z=Z.int()), 'expomf_half_epoch: Z must be float32, got torch.int32', False),
        (half(Z=Z[:, :2]), 'X and Z must be 2-D tables of one width', False),
        (half(X=torch.zeros(5, 129, device=device), Z=torch.zeros(4, 129, device=device)),
         r'd=129 unsupported \(1..128\)', False),
        (half(Z=X, mu=mx, by_row=True), 'X and Z must be different tables', False),
        (half(mu=mx), r'mu indexed by column needs 4 entries', False),
        (half(by_row=True), r'mu indexed by row needs 5 entries', False),
        (half(mu=mz.double()), 'mu must be float32', False),
        (half(mu=mx, by_row=True, mu_out=mx), 'mu_out must be a buffer of its own', False),
        (half(mu_out=torch.empty(5, device=device)), r'mu_out and mu need one float32 entry per row \(5\)', False),
        (half(rowptr=rp[:-1]), 'rowptr needs 6 entries', False),
        (half(order=torch.arange(6, dtype=torch.int32, device=device)), 'row_order must be a list of at most 5 rows',
         False),
        (half(cols=cl.long()), 'cols must be torch.int32', False),
        (half(order=order.long()), 'row_order must be torch.int32', False),
        (half(cols=cl[:-1]), r'rowptr must rise from 0 to len\(cols\) = 6', True),
        (half(cols=cl + 4), r'a column is outside \[0, 4\)', True),
        (half(order=order + 1), r'a row of row_order is outside \[0, 5\)', True),
    ]


def serec_cases(torch, device):
    from qrec_b200 import engine as E
    X, Z, rp, cl, order = _exposure_problem(torch, device)
    irp, icl = (_t(torch, device, a) for a in _csr([[0, 3], [1, 3], [0, 4], [3]]))
    iorder = torch.arange(4, dtype=torch.int32, device=device)
    A = torch.full((4,), 0.5, dtype=torch.float64, device=device)
    deg = torch.ones(5, dtype=torch.int32, device=device)

    def half(X=X, Z=Z, rowptr=rp, cols=cl, asum=A, deg=deg, row_is_user=True, order=order, **kw):
        return lambda: E.serec_half_epoch(X, Z, rowptr, cols, asum, deg, row_is_user, 1e-3, 0.01, order, **kw)

    out = torch.empty(4, dtype=torch.float64, device=device)
    items = dict(X=Z, Z=X, rowptr=irp, cols=icl, row_is_user=False, order=iorder)
    return [
        (half(X=X.double(), Z=Z.double()), 'serec_half_epoch: X must be float32, got torch.float64', False),
        (half(Z=Z[:, :2]), 'X and Z must be 2-D tables of one width', False),
        (half(X=torch.zeros(5, 129, device=device), Z=torch.zeros(4, 129, device=device)),
         r'd=129 unsupported \(1..128\)', False),
        (half(Z=X), 'X and Z must be different tables', False),
        (half(asum=A.float()), r'asum needs one float64 entry per item \(4\)', False),
        (half(asum=torch.zeros(5, dtype=torch.float64, device=device)), r'asum needs one float64 entry per item \(4\)',
         False),
        (half(deg=deg.long()), r'deg needs one int32 entry per user \(5\)', False),
        (half(deg=torch.cat([deg, deg])), r'deg needs one int32 entry per user \(5\)', False),
        (half(asum_out=A, **items), 'asum_out must be a buffer of its own', False),
        (half(asum_out=out.float(), **items), r'asum_out needs one float64 entry per row \(4\)', False),
        (half(asum_out=torch.empty(5, dtype=torch.float64, device=device)), 'the rows must be the items', False),
        (half(rowptr=rp[:-1]), 'rowptr needs 6 entries', False),
        (half(cols=cl.long()), 'cols must be torch.int32', False),
        (half(deg=deg - 2), 'serec_half_epoch: deg must not be negative', True),
        (half(cols=cl[:-1]), r'rowptr must rise from 0 to len\(cols\) = 6', True),
        (half(cols=cl + 4), r'a column is outside \[0, 4\)', True),
        (half(order=order + 1), r'a row of row_order is outside \[0, 5\)', True),
    ]


def cofactor_cases(torch, device):
    from qrec_b200 import engine as E
    n_items, n_users, d = 4, 5, 3
    f64 = torch.float64
    Y, G = torch.rand(n_items, d, dtype=f64, device=device), torch.rand(n_items, d, dtype=f64, device=device)
    X = torch.rand(n_users, d, dtype=f64, device=device)
    w, c = torch.zeros(n_items, dtype=f64, device=device), torch.zeros(n_items, dtype=f64, device=device)
    XtX = X.T @ X
    irp, icol = (_t(torch, device, a) for a in _csr([[0, 3], [1], [2, 4], [0]]))
    srp, scol = (_t(torch, device, a) for a in _csr([[1], [0, 2], [1], []]))
    item_csr = (irp, icol, torch.ones(icol.shape[0], dtype=f64, device=device))
    sppmi = (srp, scol, torch.ones(scol.shape[0], dtype=f64, device=device))

    def sweep(Y=Y, G=G, w=w, c=c, X=X, XtX=XtX, item_csr=item_csr, sppmi=sppmi, **kw):
        return lambda: E.cofactor_item_sweep(Y, G, w, c, X, XtX, item_csr, sppmi, 1.0, 1.0, 10.0, **kw)

    stamps = torch.ones(n_items, dtype=torch.int32, device=device)
    return [
        (sweep(Y=Y.int()), 'Y must be float32 or float64', False),
        (sweep(G=G[:, :2]), 'G must have the shape of Y and X its width', False),
        (sweep(X=X[:, :2]), 'G must have the shape of Y and X its width', False),
        (sweep(w=w[:-1]), 'w and c need one entry per item', False),
        (sweep(XtX=XtX[:2]), r'XtX must be \[3, 3\]', False),
        (sweep(item_csr=(irp[:-1],) + item_csr[1:]), 'item and SPPMI rowptrs need 5 entries', False),
        (sweep(sppmi=sppmi[:2] + (sppmi[2][:-1],)), 'cols and vals differ in length', False),
        (sweep(stamps=stamps[:-1], sweep=2), r'stamps must hold 1 \(sweep - 1\) for every item', False),
        (sweep(stamps=stamps, sweep=3), r'stamps must hold 2 \(sweep - 1\) for every item', True),
    ]


def _knn_problem(torch, device):
    """Three rows over four columns, their float64 values and squares, and a query list with a cold query."""
    rowptr, cols = _csr([[1, 0], [2], [3, 1, 0]])
    vals = _t(torch, device, [3.0, 4.0, 2.0, 1.0, 5.0, 2.0], torch.float64)
    return dict(rowptr=_t(torch, device, rowptr), cols=_t(torch, device, cols), vals=vals, sq=vals * vals,
                means=_t(torch, device, [3.5, 2.0, 8.0 / 3], torch.float64),
                queries=_t(torch, device, [2, -1, 0], torch.int32))


def knn_neighbours_cases(torch, device):
    from qrec_b200 import engine as E
    p = _knn_problem(torch, device)

    def nb(metric=0, K=2, **kw):
        a = dict(p, **kw)
        return lambda: E.knn_neighbours(a['rowptr'], a['cols'], a['vals'], a['sq'], a['means'], 4, a['queries'],
                                        metric, K)

    bad_rp = p['rowptr'].clone()
    bad_rp[1] = 4
    return [
        (nb(metric=3), 'metric must be 0 .pcc., 1 .cos. or 2 .euclidean.', False),
        (nb(K=-1), 'K must be an integer >= 0', False),
        (nb(K=1.5), 'K must be an integer >= 0', False),
        (nb(rowptr=p['rowptr'].int()), r'rowptr must be a 1-D int64 tensor of n_rows \+ 1 entries', False),
        (nb(cols=p['cols'].long()), 'cols must be a 1-D int32 tensor', False),
        (nb(vals=p['vals'].float()), r'vals must be float64 \[6\]', False),
        (nb(sq=p['sq'][:5]), r'sq must be float64 \[6\]', False),
        (nb(means=p['means'][:2]), r'means must be float64 \[3\]', False),
        (nb(queries=p['queries'].long()), 'queries must be a 1-D int32 tensor', False),
        (nb(cols=p['cols'] + 4), r'a column is outside \[0, 4\)', True),
        (nb(queries=p['queries'] + 3), r'a query is outside \[0, 3\) and not -1 \(cold\)', True),
        (nb(queries=_t(torch, device, [0, 0], torch.int32)), 'a row is queried twice', True),
        (nb(rowptr=bad_rp), r'rowptr must rise from 0 to len\(cols\) = 6', True),
    ]


def knn_predict_cases(torch, device):
    from qrec_b200 import engine as E
    p = _knn_problem(torch, device)
    scols, svals = E.knn_sorted_view(p['rowptr'], p['cols'], p['vals'])
    i32 = torch.int32
    ids = _t(torch, device, [[0, 1], [2, -2], [1, -1]], i32)
    sims = torch.zeros(3, 2, dtype=torch.float64, device=device)
    counts = _t(torch, device, [2, 2, 1], i32)
    qpos, probe = _t(torch, device, [0, 2, 1], i32), _t(torch, device, [1, -1, 3], i32)

    def pr(sorted_cols=scols, queries=p['queries'], ids=ids, counts=counts, line_qpos=qpos, line_probe=probe, **kw):
        a = dict(p, **kw)
        return lambda: E.knn_predict(a['rowptr'], sorted_cols, svals, a['means'], 3.0, queries, ids, sims, counts,
                                     line_qpos, line_probe, True)

    return [
        (pr(means=p['means'].float()), r'means must be float64 \[3\]', False),
        (pr(queries=p['queries'].long()), 'queries must be a 1-D int32 tensor', False),
        (pr(ids=ids[:2]), r'ids / sims must be \[3, K\] and counts \[3\]', False),
        (pr(counts=counts[:2]), r'ids / sims must be \[3, K\] and counts \[3\]', False),
        (pr(line_qpos=qpos.long()), 'line_qpos and line_probe must be int32 of one length', False),
        (pr(line_probe=probe[:2]), 'line_qpos and line_probe must be int32 of one length', False),
        (pr(ids=ids.long()), 'ids must be torch.int32', False),
        (pr(line_qpos=_t(torch, device, [0, 3, 1], i32)), r'a line query position is outside \[0, 3\)', True),
        (pr(counts=counts + 2), r'a count is outside \[0, 2\]', True),
        (pr(ids=ids + 3), r'a neighbour id is outside \[0, 3\)', True),
        (pr(sorted_cols=p['cols']), 'sorted_cols must rise strictly within each row', True),
        (pr(line_probe=probe - 2), 'a probe id is below -1', True),
    ]


def slopeone_cases(torch, device):
    from qrec_b200 import engine as E
    i32, f64 = torch.int32, torch.float64
    irp, iu = (_t(torch, device, a) for a in _csr([[0, 1], [1], [0, 2]]))       # 3 items, 3 users
    urp, ui = (_t(torch, device, a) for a in _csr([[0, 2], [0, 1], [2]]))
    iv, uv = torch.ones(5, dtype=f64, device=device), torch.ones(5, dtype=f64, device=device)
    im, um = torch.ones(3, dtype=f64, device=device), torch.ones(3, dtype=f64, device=device)
    test_items = _t(torch, device, [1, -1, 2], i32)
    qpos, users = _t(torch, device, [0, 1, 2, 0], i32), _t(torch, device, [2, 0, -1, 1], i32)

    def so(item_users=iu, item_vals=iv, item_means=im, test_items=test_items, line_qpos=qpos, line_user=users):
        return lambda: E.slopeone_predict(irp, item_users, item_vals, item_means, urp, ui, uv, um, 3.0, test_items,
                                          line_qpos, line_user)

    return [
        (so(item_users=iu.long()), 'slopeone_predict: item rows: cols must be a 1-D int32 tensor', False),
        (so(item_users=iu[:4]), 'the item and user rows hold different numbers of ratings', False),
        (so(item_vals=iv.float()), r'item_vals must be float64 \[5\]', False),
        (so(item_means=im[:2]), r'item_means must be float64 \[3\]', False),
        (so(test_items=test_items.long()), 'slopeone_predict: queries must be a 1-D int32 tensor', False),
        (so(line_user=users[:3]), 'line_qpos and line_user must be int32 of one length', False),
        (so(line_qpos=qpos.long()), 'line_qpos and line_user must be int32 of one length', False),
        (so(line_user=users - 3), r'a user is outside \[0, 3\) and not -1 \(cold\)', True),
        (so(line_qpos=qpos + 3), r'a line position is outside \[0, 3\)', True),
        (so(test_items=_t(torch, device, [1, 1, 2], i32)), 'a row is queried twice', True),
        (so(item_users=iu + 3), r'item rows: a column is outside \[0, 3\)', True),
    ]


CASES = [expomf_cases, serec_cases, cofactor_cases, knn_neighbours_cases, knn_predict_cases, slopeone_cases]


@pytest.mark.parametrize('cases', CASES, ids=[f.__name__ for f in CASES])
def test_checks_on_cpu_tensors(cases):
    import torch
    check_cases(cases(torch, 'cpu'), on_device=False)


def test_valid_calls_stop_at_the_device_check():
    """Calls whose shapes, lengths and dtypes are valid get as far as the device check on CPU tensors."""
    import torch
    from qrec_b200 import engine as E
    X, Z, rp, cl, order = _exposure_problem(torch, 'cpu')
    irp, icl = (torch.from_numpy(a) for a in _csr([[0, 3], [1, 3], [0, 4], [3]]))
    f64 = torch.float64
    A, deg = torch.full((4,), 0.5, dtype=f64), torch.ones(5, dtype=torch.int32)
    p = _knn_problem(torch, 'cpu')
    n_items, d = 4, 3
    Y, G, Xc = torch.rand(n_items, d, dtype=f64), torch.rand(n_items, d, dtype=f64), torch.rand(5, d, dtype=f64)
    crp, ccol = (torch.from_numpy(a) for a in _csr([[0, 3], [1], [2, 4], [0]]))
    srp, scol = (torch.from_numpy(a) for a in _csr([[1], [0, 2], [1], []]))
    cof = (Y, G, torch.zeros(n_items, dtype=f64), torch.zeros(n_items, dtype=f64), Xc, Xc.T @ Xc,
           (crp, ccol, torch.ones(ccol.shape[0], dtype=f64)), (srp, scol, torch.ones(scol.shape[0], dtype=f64)))
    calls = [
        lambda: E.expomf_half_epoch(X, Z, rp, cl, torch.full((4,), 0.1), False, 1e-5, 1.0, order),
        lambda: E.serec_half_epoch(X, Z, rp, cl, A, deg, True, 1e-3, 0.01, order),
        lambda: E.serec_half_epoch(Z, X, irp, icl, A, deg, False, 1e-3, 0.01, torch.arange(4, dtype=torch.int32),
                                   asum_out=torch.empty(4, dtype=f64)),
        lambda: E.cofactor_item_sweep(*cof, 1.0, 1.0, 10.0),
        lambda: E.cofactor_item_sweep(*cof, 1.0, 1.0, 10.0, stamps=torch.ones(n_items, dtype=torch.int32), sweep=2),
        lambda: E.knn_neighbours(p['rowptr'], p['cols'], p['vals'], p['sq'], p['means'], 4, p['queries'], 0, 2),
    ]
    for call in calls:
        with pytest.raises(E.QRecError, match=CUDA):
            call()


def test_svdpp_checks():
    import torch
    from qrec_b200 import engine as E
    U, I, d = 4, 3, 2
    f64 = torch.float64
    tabs = dict(P=torch.rand(U, d, dtype=f64), Q=torch.rand(I, d, dtype=f64), Y=torch.rand(I, d, dtype=f64),
                Bu=torch.zeros(U, dtype=f64), Bi=torch.zeros(I, dtype=f64))
    rowptr, cols = (torch.from_numpy(a) for a in _csr([[0, 1], [2], [], [0]]))
    u, i, r = torch.tensor([0, 1], dtype=torch.int32), torch.tensor([1, 2], dtype=torch.int32), torch.ones(2, dtype=f64)
    loss = torch.zeros(1, dtype=f64)

    def ordered(u=u, rowptr=rowptr, **kw):
        t = dict(tabs, **kw)
        return lambda: E.svdpp_sgd_ordered(t['P'], t['Q'], t['Y'], t['Bu'], t['Bi'], u, i, r, rowptr, cols, 0.01, 0.1,
                                           0.1, 0.1, 0.1, 3.0, loss)

    f32tabs = {k: v.float() for k, v in tabs.items()}
    order = torch.arange(U, dtype=torch.int32)

    def fast(vals=torch.ones(cols.shape[0]), rowptr=rowptr, **kw):
        t = dict(f32tabs, **kw)
        return lambda: E.svdpp_epoch_usermajor(t['P'], t['Q'], t['Y'], t['Bu'], t['Bi'], rowptr, cols, vals, order,
                                               0.01, 0.1, 0.1, 0.1, 0.1, 3.0, loss)

    check_cases([
        (ordered(P=tabs['P'].int()), 'P must be float32 or float64, got torch.int32', False),
        (ordered(u=u[:1]), 'svdpp_sgd_ordered: u, i, r differ in length', False),
        (ordered(rowptr=rowptr[:-1]), 'svdpp_sgd_ordered: rowptr has 4 entries for 4 users', False),
        (ordered(Y=tabs['Y'][:, :1]), 'svdpp: P, Q, Y must be 2-D tables of one width', False),
        (ordered(Y=tabs['Y'][:2]), 'svdpp: Y / Bi need one row per item of Q, Bu one per user of P', False),
        (ordered(Bu=tabs['Bu'][:3]), 'svdpp: Y / Bi need one row per item of Q, Bu one per user of P', False),
        (ordered(), CUDA, False),
        (fast(vals=torch.ones(cols.shape[0] + 1)), 'svdpp_epoch_usermajor: cols and vals differ in length', False),
        (fast(rowptr=rowptr[:-1]), 'svdpp_epoch_usermajor: rowptr has 4 entries for 4 users', False),
        (fast(Q=f32tabs['Q'][:, :1]), 'svdpp: P, Q, Y must be 2-D tables of one width', False),
        (fast(Bi=f32tabs['Bi'][:2]), 'svdpp: Y / Bi need one row per item of Q, Bu one per user of P', False),
        (fast(), CUDA, False),
    ], on_device=False)


def test_wrmf_checks():
    import torch
    from qrec_b200 import engine as E
    X, Z = torch.rand(4, 3, dtype=torch.float64), torch.rand(5, 3, dtype=torch.float64)
    rowptr, cols = (torch.from_numpy(a) for a in _csr([[0, 1], [2], [], [4]]))
    vals = torch.ones(cols.shape[0], dtype=torch.float64)
    G = Z.T @ Z
    order = torch.arange(4, dtype=torch.int32)
    check_cases([
        (lambda: E.als_gram(Z.int()), 'Z must be float32 or float64', False),
        (lambda: E.als_gram(Z), CUDA, False),
        (lambda: E.als_solve_rows(X.int(), Z, G, rowptr, cols, vals, 1.0, 1.0, order), 'X must be float32 or float64',
         False),
        (lambda: E.als_solve_rows(X, Z[:, :2], G, rowptr, cols, vals, 1.0, 1.0, order),
         r'X and Z differ in width \(3, 2\)', False),
        (lambda: E.als_solve_rows(X, Z, G, rowptr, cols, vals, 1.0, 1.0, order), CUDA, False),
    ], on_device=False)


def test_knn_sorted_view_stays_on_the_host():
    """knn_sorted_view launches no kernel: it takes CPU tensors and checks their contents itself."""
    import torch
    from qrec_b200 import engine as E
    p = _knn_problem(torch, 'cpu')
    scols, svals = E.knn_sorted_view(p['rowptr'], p['cols'], p['vals'])
    assert scols.tolist() == [0, 1, 2, 0, 1, 3] and svals.tolist() == [4.0, 3.0, 2.0, 2.0, 5.0, 1.0]
    twice = torch.tensor([1, 1, 2, 3, 1, 0], dtype=torch.int32)
    check_cases([
        (lambda: E.knn_sorted_view(p['rowptr'], twice, p['vals']), 'a row lists the same column twice', False),
        (lambda: E.knn_sorted_view(p['rowptr'], p['cols'], p['vals'][:5]), r'vals must be float64 \[6\]', False),
        (lambda: E.knn_sorted_view(p['rowptr'][:-1], p['cols'], p['vals']), 'rowptr must rise from 0 to len.cols. = 6',
         False),
    ], on_device=False)


def test_knn_pair_similarity_names_both_column_arrays():
    import torch
    from qrec_b200 import engine as E
    p = _knn_problem(torch, 'cpu')
    scols, svals = E.knn_sorted_view(p['rowptr'], p['cols'], p['vals'])
    _, ssq = E.knn_sorted_view(p['rowptr'], p['cols'], p['sq'])
    ab, w = torch.tensor([0, 2], dtype=torch.int32), torch.tensor([0.5, 1.0], dtype=torch.float64)
    check_cases([
        (lambda: E.knn_pair_similarity(p['rowptr'], p['cols'].long(), p['vals'], p['sq'], p['means'], scols, svals,
                                       ssq, ab, ab, w), 'cols and sorted_cols must be 1-D int32 tensors of one length',
         False),
        (lambda: E.knn_pair_similarity(p['rowptr'], p['cols'], p['vals'], p['sq'], p['means'], scols, svals, ssq, ab,
                                       ab, w), CUDA, False),
    ], on_device=False)
