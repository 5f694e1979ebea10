"""Every (NT, ngroups) class of the ALS-family row solves against float64 references (als_shape_cases.py): the Gram,
the WRMF row solve, the CoFactor item sweep and the exposure solve of ExpoMF and SERec, at every width of the table.

The Gram and the WRMF loss are exact on integer inputs and compared bit for bit.  Solved rows are judged per row,
relative to the row's |x|_inf: WRMF's within C_SOLVE d 2^-53 kappa_inf(A) (+ 2^-24 for float32 tables) of the refined
solution, the others within als_shape_cases.BOUNDS units of d 2^-53 kappa_inf(A) (+ 2^-24).  Each test rebuilds its
reference with every defect of als_shape_cases.DEFECTS that touches the case and asserts that it lies at least 10
bounds away.  Rows a row order does not name, items without contexts and rows of a failing system keep their bits."""
import numpy as np
import pytest

import als_shape_cases as R

pytestmark = pytest.mark.gpu

GAMMA = 1.0


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def E():
    from qrec_b200 import engine
    return engine


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def untouched(got, init, rows):
    keep = np.ones(len(init), bool)
    keep[np.asarray(rows, np.int64)] = False
    assert R.same_bits(got[keep], init[keep]), 'rows the launch does not name were written'


def defect_distances(ref, units, bad_of, lengths, d, defects=R.DEFECTS):
    return {k: R.worst(R.row_errors(bad_of(k), ref), units) for k in defects if R.applies(k, lengths, d)}


# ------------------------------------------------------------------------------------------------------- Gram
@pytest.mark.parametrize('d', R.WIDTHS)
def test_gram(torch, E, d):
    for n in R.GRAM_SIZES:
        Z = R.gram_case(d, n)
        Zi = Z.astype(np.int64)
        ref = (Zi.T @ Zi).astype(np.float64)
        for dt in (np.float32, np.float64):
            G = host(E.als_gram(dev(Z.astype(dt))))
            assert R.same_bits(G, ref), 'als_gram d=%d n=%d %s' % (d, n, dt.__name__)
            assert R.same_bits(G, np.ascontiguousarray(G.T))


# ------------------------------------------------------------------------------------------------------- WRMF
SOLVE = [(d, s) for d in R.WIDTHS for s in ('tails', 'many') if s == 'tails' or d in R.CLASS_WIDTHS]


def _solve(torch, E, c, X0, dt, order, lam=R.LAM):
    X, Z = dev(X0), dev(c['Z'].astype(dt))
    loss = torch.zeros(1, dtype=torch.float64, device='cuda')
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    E.als_solve_rows(X, Z, E.als_gram(Z), dev(c['rowptr']), dev(c['cols']), dev(c['vals'].astype(dt)), lam, R.ALPHA,
                     dev(order), loss=loss, n_failed=n_failed)
    return host(X), loss.item(), int(n_failed.item())


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('d,structure', SOLVE, ids=['d%d-%s' % k for k in SOLVE])
def test_solve_rows(torch, E, d, structure, dtype):
    c = R.solve_case(d, structure)
    dt = np.dtype(dtype).type
    X0 = c['X'].astype(dt)
    got, loss, failed = _solve(torch, E, c, X0, dt, c['order'])
    assert failed == 0 and loss == float(R.solve_loss(c)), 'the loss of integer inputs is exact'
    untouched(got, X0, c['order'])
    again, loss2, _ = _solve(torch, E, c, X0, dt, c['order'][::-1].copy())
    assert R.same_bits(again, got) and loss2 == loss, 'a reversed row order changed the bits'
    ref, kap = R.solve_reference(d, structure)
    units = R.solve_units(d, kap, dtype == 'float32', R.C_SOLVE)
    lengths = np.diff(c['rowptr'])[c['order']]
    R.judge('als_solve_rows %s d=%d %s' % (dtype, d, structure), {'X': 1.0}, {
        'X': (R.worst(R.row_errors(got[c['order']], ref), units),
              defect_distances(ref, units, lambda k: R.solve_reference(d, structure, k)[0], lengths, d))})


@pytest.mark.parametrize('d', R.CLASS_WIDTHS)
def test_solve_rows_all_failing(torch, E, d):
    """lambda = -1e9: no row's system is positive definite; every failure is counted and every row keeps its bits."""
    c = R.solve_case(d, 'tails')
    for dt in (np.float32, np.float64):
        X0 = c['X'].astype(dt)
        got, _, failed = _solve(torch, E, c, X0, dt, c['order'], lam=-1e9)
        assert failed == len(c['order']) and R.same_bits(got, X0)


# ------------------------------------------------------------------------------------------------------- CoFactor
def _sweep(torch, E, c, dt, gamma):
    Y, G, w, cc, X = (dev(c[k]) for k in ('Y', 'G', 'w', 'c', 'X'))
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    E.cofactor_item_sweep(Y, G, w, cc, X, E.als_gram(X), tuple(dev(a) for a in c['item_csr']),
                          tuple(dev(a) for a in c['sppmi']), R.LAM, gamma, R.ALPHA, n_failed=n_failed)
    return [host(t) for t in (Y, G, w, cc)], int(n_failed.item())


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('d', R.WIDTHS)
def test_cofactor_item_sweep(torch, E, d, dtype):
    c = R.cofactor_case(d, dtype)
    f32 = dtype == 'float32'
    (Y, G, w, cc), failed = _sweep(torch, E, c, dtype, GAMMA)
    again, _ = _sweep(torch, E, c, dtype, GAMMA)
    assert failed == 0 and all(R.same_bits(a, b) for a, b in zip(again, (Y, G, w, cc))), 'two sweeps differ'
    srp = c['sppmi'][0]
    has = np.diff(srp) > 0
    for got, init in ((G, c['G']), (w, c['w']), (cc, c['c'])):
        assert R.same_bits(got[~has], init[~has]), 'an item without contexts changed G, w or c'
    ref = R.cofactor_reference(c, R.LAM, GAMMA)
    rY, rG, rw, rc = ref[:4]
    uY, uG, uw, uc = R.cofactor_units(c, ref, f32)
    bads = {k: R.cofactor_reference(c, R.LAM, GAMMA, k) for k in R.DEFECTS
            if R.applies(k, list(np.diff(srp)) + list(np.diff(c['item_csr'][0])), d)}

    def scalar(a, r, u):
        return R.worst(np.abs(np.asarray(a, np.float64) - r)[has], u[has])
    R.judge('cofactor_item_sweep %s d=%d' % (dtype, d), R.BOUNDS['cofactor_' + ('f32' if f32 else 'f64')], {
        'Y': (R.worst(R.row_errors(Y, rY), uY), {k: R.worst(R.row_errors(b[0], rY), uY) for k, b in bads.items()}),
        'G': (R.worst(R.row_errors(G[has], rG[has]), uG[has]),
              {k: R.worst(R.row_errors(b[1][has], rG[has]), uG[has]) for k, b in bads.items()}),
        'w': (scalar(w, rw, uw), {k: scalar(b[2], rw, uw) for k, b in bads.items() if k in ('drop_last', 'column')}),
        'c': (scalar(cc, rc, uc), {k: scalar(b[3], rc, uc) for k, b in bads.items() if k in ('drop_last', 'column')})})
    # gamma = -1e9: every G system fails inside the one launch, next to Y systems that solve
    (_, Gf, _, _), failed = _sweep(torch, E, c, dtype, -1e9)
    assert failed == int(has.sum()) and R.same_bits(Gf, c['G'])


# ------------------------------------------------------------------------------------------------------- exposure
EXPO = SOLVE


def _expo(torch, E, c, call, max_ctas):
    """Runs one exposure half on fresh copies; returns (X, fused output or None)."""
    X, Z = dev(c['X']), dev(c['Z'])
    n_failed = torch.zeros(1, dtype=torch.int32, device='cuda')
    args = dict(n_failed=n_failed, max_ctas=max_ctas)
    csr = dev(c['rowptr']), dev(c['cols'])
    out = None
    if call[0] == 'expomf':
        item = call[1] == 'item'
        if item:
            out = torch.full((len(c['X']),), 7.0, device='cuda')
        E.expomf_half_epoch(X, Z, *csr, dev(c['mu_x'] if item else c['mu_z']), item, R.LAM, R.LAM_Y,
                            dev(c['order']), mu_out=out, **args)
    else:
        _, row_is_user, given = call
        asum = dev(c['asum_z'] if row_is_user else c['asum_x']) if given else None
        if not row_is_user:
            out = torch.full((len(c['X']),), 7.0, dtype=torch.float64, device='cuda')
        E.serec_half_epoch(X, Z, *csr, asum, dev(c['deg_x'] if row_is_user else c['deg_z']), row_is_user, R.LAM,
                           R.LAM_Y, dev(c['order']), asum_out=out, mu0=R.SO.MU0, **args)
    assert int(n_failed.item()) == 0
    return host(X), (None if out is None else host(out))


EXPO_CALLS = [('expomf', 'user'), ('expomf', 'item'), ('serec', True, False), ('serec', True, True),
              ('serec', False, False), ('serec', False, True)]


@pytest.mark.parametrize('call', EXPO_CALLS, ids=['expomf-user', 'expomf-item', 'serec-user-uniform', 'serec-user',
                                                  'serec-item-uniform', 'serec-item'])
@pytest.mark.parametrize('d,structure', EXPO, ids=['d%d-%s' % k for k in EXPO])
def test_exposure_half(torch, E, d, structure, call):
    c = R.exposure_case(d, structure)
    got, out = _expo(torch, E, c, call, 0)
    if structure == 'tails':
        for k in (1, 7):
            g2, o2 = _expo(torch, E, c, call, k)
            assert R.same_bits(g2, got) and (out is None or R.same_bits(o2, out)), 'max_ctas=%d changed the bits' % k
    untouched(got, c['X'], c['order'])
    if out is not None:
        untouched(out, np.full(len(out), 7.0, out.dtype), c['order'])
    if call[0] == 'expomf':
        M, lam_y, fam = R.exposure_prior(c, 'expomf_' + call[1], True), R.LAM_Y, 'expomf'
    else:
        M, lam_y, fam = R.exposure_prior(c, 'serec', call[2], call[1]), R.LAM_Y, 'serec'
    ref, kap = R.exposure_reference(c, M, R.LAM, lam_y)
    units = R.solve_units(d, kap, True)
    lengths = list(np.diff(c['rowptr'])[c['order']]) + [len(c['Z'])]
    outputs = {'X': (R.worst(R.row_errors(got[c['order']], ref), units),
                     defect_distances(ref, units, lambda k: R.exposure_reference(c, M, R.LAM, lam_y, k)[0], lengths,
                                      d))}
    if out is not None:
        n_z = len(c['Z'])

        def fused(k=None):
            s = R.exposure_sums(c, got, M, lam_y, k)
            return (1.0 + s - 1.0) / (1.0 + 99.0 + n_z - 2) if fam == 'expomf' else s
        unit = R.U32 if fam == 'expomf' else n_z * R.U64
        r = fused()

        def rel(a):
            return float((np.abs(np.asarray(a, np.float64) - r) / (unit * np.abs(r))).max())
        outputs['mu_out' if fam == 'expomf' else 'asum_out'] = (
            rel(out[c['order']]), {k: rel(fused(k)) for k in ('drop_last', 'column')})
    R.judge('%s d=%d %s' % ('-'.join(map(str, call)), d, structure), R.BOUNDS[fam], outputs)
