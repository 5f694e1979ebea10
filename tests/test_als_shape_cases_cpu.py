"""The cases of test_gpu_als_shape_matrix.py checked without a GPU: the width table reaches every (NT, ngroups) class of
the ALS-family row solves at both ends and every d mod 4 at both NT (through the header's own tile functions, built
for the host); the builders reach every length and size edge they are named for; the integer inputs keep every sum
exact; the references agree with the oracles; the device's own step source (als_step.cuh) lies inside the WRMF bound
on every case; and every defective reference lies at least TEETH bounds outside."""
import numpy as np
import pytest

import als_shape_cases as R
from test_wrmf_cpu import host, host_side  # noqa: F401

def test_tile_restatement_is_the_header(host):  # noqa: F811
    assert (host.host_als_threads(), host.host_als_stage(), host.host_als_gram_chunk(), host.host_als_max_d()) == \
        (R.THREADS, R.STAGE, R.GRAM_CHUNK, R.MAX_D)
    for d in range(1, R.MAX_D + 1):
        nt = host.host_als_tiles_per_thread(d)
        assert (host.host_als_pad4(d), host.host_als_tiles_of(d), nt, host.host_als_groups(nt, d)) == \
            (R.pad4(d), R.tiles_of(d), R.tiles_per_thread(d), R.groups(d))


def test_widths_reach_every_class_at_both_ends(host):  # noqa: F811
    cls = {}
    for d in range(1, R.MAX_D + 1):
        nt = host.host_als_tiles_per_thread(d)
        cls.setdefault((nt, host.host_als_groups(nt, d)), []).append(d)
    assert len(cls) == 13
    for k, ds in cls.items():
        assert ds == list(range(ds[0], ds[-1] + 1))                 # every class is one run of widths
        assert ds[0] in R.WIDTHS and ds[-1] in R.WIDTHS, k
    assert {R.tile_class(d) for d in R.CLASS_WIDTHS} == set(cls) and len(R.CLASS_WIDTHS) == 13
    for nt in (1, 3):
        assert {d % 4 for d in R.WIDTHS if R.tiles_per_thread(d) == nt} == {0, 1, 2, 3}
    assert {88, 89, 96, 97} <= set(R.WIDTHS) and R.tile_class(88)[0] == 1 and R.tile_class(89)[0] == 3
    assert any(97 <= d <= 127 for d in R.WIDTHS)                     # warp 0's fourth register partly filled
    assert max(R.WIDTHS) == R.MAX_D and len(R.WIDTHS) == 40


def _lengths(c):
    return np.diff(c['rowptr'])


def test_builders_reach_every_edge():
    for d in R.WIDTHS:
        g = R.groups(d)
        for build in (R.solve_case, R.exposure_case):
            c = build(d, 'tails')
            ln = _lengths(c)
            assert {0, 1, g - 1, g, g + 1, 31, 32, 33, 63, 64, 65} <= set(ln.tolist()) and ln.max() > 1024
            order = c['order']
            assert len(np.unique(order)) == len(order) == len(ln) - R.UNNAMED
            assert (ln[np.setdiff1d(np.arange(len(ln)), order)] > 0).all()        # unnamed rows have entries
            assert np.all(np.diff(ln[order]) <= 0)
        for build in (R.solve_case, R.exposure_case):
            c = build(d, 'tails')
            assert all(len(np.unique(c['cols'][a:b])) == b - a for a, b in zip(c['rowptr'][:-1], c['rowptr'][1:]))
        cf = R.cofactor_case(d, 'float64')
        srp, scol, sval = cf['sppmi']
        ctx_len = set(np.diff(srp).tolist())
        assert {0, 1, g, 31, 32, 33, 65} == ctx_len
        assert set(np.diff(cf['item_csr'][0]).tolist()) == ctx_len
        n = len(srp) - 1
        M = np.zeros((n, n))
        M[np.repeat(np.arange(n), np.diff(srp)), scol] = sval
        assert np.array_equal(M, M.T) and not np.diag(M).any()                    # symmetric, no self-context
        row = np.repeat(np.arange(n), np.diff(srp))
        assert (scol < row).any() and (scol > row).any()
        assert all(np.all(np.diff(scol[a:b]) > 0) for a, b in zip(srp[:-1], srp[1:]))
    for d in R.CLASS_WIDTHS:
        for build in (R.solve_case, R.exposure_case):
            assert len(build(d, 'many')['order']) > R.SMS * R.MAX_PER_SM
    chunk = R.GRAM_CHUNK
    assert {0, 1, 31, 32, 33, chunk - 1, chunk, chunk + 1} <= set(R.GRAM_SIZES)
    assert max(R.GRAM_SIZES) > 3 * chunk and max(R.GRAM_SIZES) % R.STAGE != 0
    for s in ('tails', 'many'):
        assert {R.expo_rows(d, s) % 32 for d in R.WIDTHS} == {0, 1, 31}
        assert {R.expo_rows(d, s) % 32 for d in R.CLASS_WIDTHS} == {0, 1, 31}


def test_integer_inputs_keep_every_sum_exact():
    lim = 2.0 ** 53
    for d in R.WIDTHS:
        for n in R.GRAM_SIZES:
            Z = np.abs(R.gram_case(d, n))
            assert (Z.T @ Z).max(initial=0) < lim and np.array_equal(Z, np.round(Z)) and Z.max(initial=0) <= 4
        for s in ('tails', 'many'):
            c = R.solve_case(d, s)
            Z, X = np.abs(c['Z']), np.abs(c['X'])
            assert Z.max() <= 4 and X.max() <= 4 and set(np.unique(c['vals'])) <= {1.0, 2.0, 3.0, 4.0, 5.0}
            G = (Z.T @ Z).max()
            for r in c['order']:
                z = Z[c['cols'][c['rowptr'][r]:c['rowptr'][r + 1]]]
                w = R.ALPHA * c['vals'][c['rowptr'][r]:c['rowptr'][r + 1]]
                assert G + (w[:, None] * z).T.dot(z).max(initial=0) + R.LAM < lim
                assert ((1 + w)[:, None] * z).sum(0).max(initial=0) < lim
            assert sum(((1 + Z[c['cols']] @ X[r]) ** 2).sum() for r in range(len(X))) < lim


def test_wrmf_reference_is_the_oracle():
    from oracle import wrmf_oracle as W
    for d in R.CLASS_WIDTHS:
        for s in ('tails', 'many'):
            c = R.solve_case(d, s)
            ref, _ = R.solve_reference(d, s)
            X = c['X'].copy()
            loss = W.solve_side(X, c['Z'], c['rowptr'], c['cols'], c['vals'], R.LAM, R.ALPHA, rows=c['order'],
                                with_loss=True)
            np.testing.assert_allclose(ref, X[c['order']], rtol=1e-12, atol=1e-12 * np.abs(ref).max())
            assert loss == R.solve_loss(c)


def test_exposure_references_are_the_oracles():
    from oracle import expomf_oracle as EO, serec_oracle as SO
    for d in (1, 20, 97):
        c = R.exposure_case(d, 'tails')
        args = c['rowptr'], c['cols']
        for kind in ('expomf_user', 'expomf_item'):
            M = R.exposure_prior(c, kind, True)
            ref, _ = R.exposure_reference(c, M, R.LAM, 1.0)
            X = c['X'].astype(np.float64)
            EO.solve_side(X, c['Z'], *args, c['mu_x'] if kind == 'expomf_item' else c['mu_z'], kind == 'expomf_item',
                          R.LAM, 1.0, rows=c['order'])
            np.testing.assert_allclose(ref, X[c['order']], rtol=1e-11, atol=1e-12 * np.abs(ref).max())
        sums = R.exposure_sums(c, X, R.exposure_prior(c, 'expomf_item', True), 1.0)
        prior = EO.prior_rows(X, c['Z'], *args, c['mu_x'], rows=c['order'])
        np.testing.assert_allclose((1 + sums - 1) / (1 + 99 + len(c['Z']) - 2), prior, rtol=1e-13)
        for row_is_user in (True, False):
            M = R.exposure_prior(c, 'serec', True, row_is_user)
            ref, _ = R.exposure_reference(c, M, R.LAM, R.LAM_Y)
            X = c['X'].astype(np.float64)
            SO.solve_side(X, c['Z'], *args, M, R.LAM, R.LAM_Y, rows=c['order'])
            np.testing.assert_allclose(ref, X[c['order']], rtol=1e-11, atol=1e-12 * np.abs(ref).max())
        np.testing.assert_allclose(R.exposure_sums(c, X, M, R.LAM_Y),
                                   SO.asum_rows(X, c['Z'], *args, M, R.LAM_Y, rows=c['order']), rtol=1e-13)


def test_cofactor_reference_is_the_oracle():
    from oracle import cofactor_oracle as CO
    for d in (1, 20, 97):
        for dt in ('float64', 'float32'):
            c = R.cofactor_case(d, dt)
            got = R.cofactor_reference(c, R.LAM, 1.0)
            Y, G, w, cc = (np.array(c[k], copy=True) for k in ('Y', 'G', 'w', 'c'))
            CO.item_sweep(Y, G, w, cc, c['X'], c['item_csr'], c['sppmi'], R.LAM, 1.0)
            for a, b in zip(got[:4], (Y, G, w, cc)):
                assert a.dtype == b.dtype
                if dt == 'float64':
                    np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-10 * np.abs(b).max())
                else:                    # rows rounded to float32 in the same places: a few ulps at most
                    np.testing.assert_allclose(a, b, rtol=4 * R.U32, atol=4 * R.U32 * np.abs(b).max())


@pytest.mark.parametrize('d', R.WIDTHS)
def test_device_step_source_inside_and_defects_outside_the_wrmf_bound(host, d):  # noqa: F811
    """host_als_side_* (als_step.cuh's own Cholesky and substitutions) on every solve case lies within C_SOLVE units,
    so the bound is not tuned to the GPU; every defect lies at least TEETH bounds away."""
    for s in ('tails', 'many') if d in R.CLASS_WIDTHS else ('tails',):
        c = R.solve_case(d, s)
        ref, kap = R.solve_reference(d, s)
        for dt in (np.float64, np.float32):
            units = R.solve_units(d, kap, dt == np.float32, R.C_SOLVE)
            X = c['X'].astype(dt)
            loss, failed = host_side(host, X, c['Z'].astype(dt), (c['rowptr'], c['cols'], c['vals']), R.LAM,
                                     R.ALPHA, with_loss=True)
            assert failed == 0
            assert R.worst(R.row_errors(X[c['order']], ref), units) <= 1.0
            for defect in R.DEFECTS:
                if R.applies(defect, _lengths(c)[c['order']], d):
                    bad, _ = R.solve_reference(d, s, defect)
                    assert R.worst(R.row_errors(bad, ref), units) >= R.TEETH, (s, dt, defect)


@pytest.mark.parametrize('d', R.WIDTHS)
def test_exposure_and_cofactor_defects_lie_outside_their_bounds(d):
    from oracle import serec_oracle as SO
    for s in ('tails', 'many') if d in R.CLASS_WIDTHS else ('tails',):
        c = R.exposure_case(d, s)
        for kind, rows, lam_y, fam in (('expomf_user', True, 1.0, 'expomf'), ('expomf_item', True, 1.0, 'expomf'),
                                       ('serec', True, R.LAM_Y, 'serec'), ('serec', False, R.LAM_Y, 'serec')):
            M = R.exposure_prior(c, kind, True, rows)
            ref, kap = R.exposure_reference(c, M, R.LAM, lam_y)
            units = R.solve_units(d, kap, True)
            for defect in R.DEFECTS:
                if not R.applies(defect, list(_lengths(c)[c['order']]) + [len(c['Z'])], d):
                    continue
                bad, _ = R.exposure_reference(c, M, R.LAM, lam_y, defect)
                assert R.worst(R.row_errors(bad, ref), units) >= R.TEETH * R.BOUNDS[fam]['X'], (s, kind, defect)
    for dt in ('float64', 'float32'):
        c = R.cofactor_case(d, dt)
        ref = R.cofactor_reference(c, R.LAM, 1.0)
        uY, uG = R.cofactor_units(c, ref, dt == 'float32')[:2]
        has = np.diff(c['sppmi'][0]) > 0
        lengths = list(np.diff(c['sppmi'][0])) + list(np.diff(c['item_csr'][0]))
        for defect in R.DEFECTS:
            if not R.applies(defect, lengths, d):
                continue
            bY, bG = R.cofactor_reference(c, R.LAM, 1.0, defect)[:2]
            dist = max(R.worst(R.row_errors(bY, ref[0]), uY), R.worst(R.row_errors(bG[has], ref[1][has]), uG[has]))
            assert dist >= R.TEETH * R.BOUNDS['cofactor_' + ('f32' if dt == 'float32' else 'f64')]['Y'], (dt, defect)
