"""The float64 wave oracle (k1_wave_oracle.py) checked without a GPU.

The GPU tests of the user-major BPR epoch compare the kernel with wave_oracle, which is vectorised over the users of a
wave.  Here it must equal a loop written straight from the comment above bpr_sgd_usermajor_kernel (bpr_kernels.cu) and the
chunk rule of um_waves.cuh, on small epochs built to hit what vectorising could get wrong; and every case of
test_gpu_k1_matrix.py must reach the branch of the wave rule, the degrees and the lane shape it is named for."""
import math

import numpy as np
import pytest

from k1_wave_oracle import (CASES, CH, LONG_USERS, SATURATED_USER, case_data, case_launches, case_rowptr, row_lpr,
                            wave_chunks, wave_oracle)
from test_k1_schedule_cpu import chunk_rule_waves, lib  # noqa: F401


def naive_epoch(P0, Q0, rowptr, i, j, launches, lr, reg_u, reg_i, shift=0):
    """One triple at a time.  A launch is cut into chunks of CH triples and swept in waves of wave_chunks() chunks; a
    user belongs to the wave whose chunks hold its first triple.  A wave reads item rows from the table as it was when
    the wave started and adds its item-row deltas to the table afterwards; P[u] is updated after every triple."""
    P, Q = P0.astype(np.float64), Q0.astype(np.float64)
    loss = 0.0
    for ua, ub in launches:
        rp = rowptr[ua:ub + 1]
        n, trip_off = int(rp[-1] - rp[0]), int(rp[0])
        if n == 0:
            continue
        wave = wave_chunks(n, Q.shape[0], Q.shape[1])
        chunk_of, s, e = chunk_rule_waves(rp, n, trip_off, 1)          # waves of one chunk: the user's chunk
        wave_of = np.where(chunk_of >= 0, (chunk_of + shift // CH) // wave, -1)
        for w in range(int(wave_of.max()) + 1):
            Qw, deltas = Q.copy(), []
            for r in np.nonzero(wave_of == w)[0]:
                u = ua + r
                for t in range(trip_off + int(s[r]), trip_off + int(e[r])):
                    qi, qj = Qw[i[t]], Qw[j[t]]
                    sg = 1.0 / (1.0 + math.exp(-float(P[u] @ qi - P[u] @ qj)))
                    g = lr * (1.0 - sg)
                    loss -= math.log(sg)
                    pn = P[u] + g * (qi - qj)
                    deltas.append((i[t], g * (1 - lr * reg_i) * pn - lr * reg_i * qi))
                    deltas.append((j[t], -g * (1 - lr * reg_i) * pn - lr * reg_i * qj))
                    P[u] = (1 - lr * reg_u) * pn
            for row, delta in deltas:
                Q[row] += delta
    return P, Q, loss


ITEMS, D, USERS, SPLIT, LONG = 20, 8, 150, 70, 20


@pytest.fixture(scope='module')
def small():
    rng = np.random.default_rng(5)
    deg = rng.integers(0, 61, USERS)
    deg[:3] = 0; deg[-4:] = 0; deg[50:56] = 0       # runs of empty users at both ends and inside
    deg[LONG] = 200                                 # longer than two waves
    rowptr = np.zeros(USERS + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    n = int(rowptr[-1])
    i, j = rng.integers(0, ITEMS, n), rng.integers(0, ITEMS, n)
    a = int(rowptr[5])
    assert deg[5] >= 4
    i[a + 1] = i[a]                                 # an item repeated inside one user, inside one wave
    j[a + 3] = i[a]                                 # ... and as a negative of the same user
    j[a + 2] = i[a + 2]                             # i == j
    j[rowptr[LONG] + 100] = i[rowptr[LONG] + 100]
    P0, Q0 = rng.random((USERS, D)) / 3, rng.random((ITEMS, D)) / 3
    wave = wave_chunks(n, ITEMS, D)
    assert wave >= 2 and deg[LONG] > 2 * wave * CH and rowptr[SPLIT] % (wave * CH) != 0
    return rowptr, i, j, P0, Q0


@pytest.mark.parametrize('shift', [0, CH])
@pytest.mark.parametrize('launches', [[(0, USERS)], [(0, SPLIT), (SPLIT, USERS)], [(0, 2), (2, 30), (30, 31), (31, USERS)]],
                         ids=['one', 'two', 'four'])
def test_oracle_equals_the_naive_loop(small, launches, shift):
    rowptr, i, j, P0, Q0 = small
    lr, reg_u, reg_i = 0.05, 0.02, 0.07
    got = wave_oracle(P0, Q0, rowptr, i, j, launches, lr, reg_u, reg_i, shift=shift)
    ref = naive_epoch(P0, Q0, rowptr, i, j, launches, lr, reg_u, reg_i, shift=shift)
    for g, r in zip(got[:2], ref[:2]):
        np.testing.assert_allclose(g, r, rtol=1e-12, atol=0)
    assert abs(got[2] - ref[2]) <= 1e-12 * ref[2]
    # what the cases are there to tell apart does move the result; the cut launches' waves are one chunk long, and
    # moving every boundary of such a launch by a chunk regroups nobody
    others = [wave_oracle(P0, Q0, rowptr, i, j, launches, lr, reg_i, reg_u, shift=shift),
              wave_oracle(P0, Q0, rowptr, i, j, [(0, USERS)] if len(launches) > 1 else [(0, SPLIT), (SPLIT, USERS)],
                          lr, reg_u, reg_i, shift=shift)]
    if len(launches) == 1:
        others.append(wave_oracle(P0, Q0, rowptr, i, j, launches, lr, reg_u, reg_i, shift=CH - shift))
    for other in others:
        assert np.abs(other[0] - ref[0]).max() > 1e-6 and np.abs(other[1] - ref[1]).max() > 1e-6


def test_single_regulariser_is_the_default(small):
    rowptr, i, j, P0, Q0 = small
    a = wave_oracle(P0, Q0, rowptr, i, j, [(0, USERS)], 0.05, 0.02)
    b = wave_oracle(P0, Q0, rowptr, i, j, [(0, USERS)], 0.05, 0.02, 0.02)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def test_the_widths_cover_every_lane_shape():
    """lane_shape.h: LPR 4, 8, 16, 32, each with d == 4 LPR (FULL) and with idle lanes."""
    shapes = {(row_lpr(c.d // 4), c.d == 4 * row_lpr(c.d // 4)) for c in CASES if c.name.startswith('w')}
    assert shapes == {(lpr, full) for lpr in (4, 8, 16, 32) for full in (False, True)}
    for c in CASES:
        assert c.d % 4 == 0 and ('sig' not in c.entries or c.d in (16, 32, 64, 128))


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_case_reaches_its_branch(lib, case):  # noqa: F811
    rowptr = case_rowptr(case)
    deg = np.diff(rowptr)
    launches = case_launches(case, rowptr)
    assert launches[0][0] == 0 and launches[-1][1] == case.users
    assert all(a[1] == b[0] for a, b in zip(launches, launches[1:]))
    for ua, ub in launches:
        rp = rowptr[ua:ub + 1]
        n, trip_off = int(rp[-1] - rp[0]), int(rp[0])
        wave = wave_chunks(n, case.items, case.d)
        assert lib.um_wave_chunks_host(n, case.items, case.d) == wave
        assert -(-(-(-n // CH)) // wave) > 1, 'a launch of one wave'
        # the oracle's membership rule is the chunk rule
        wave_of, _, _ = chunk_rule_waves(rp, n, trip_off, wave)
        has = np.diff(rp) > 0
        np.testing.assert_array_equal(((rp[:-1] - trip_off) // (wave * CH))[has], wave_of[has])
    n = int(rowptr[-1])
    wave = wave_chunks(n, case.items, case.d)
    copy_bytes = 2 * case.items * case.d * 4
    copy_floor = 8 * copy_bytes // (24 * case.d + 12) if copy_bytes > (8 << 20) else 0
    kind = case.name.rstrip('0123456789')
    if kind == 'large':
        assert copy_floor > n // 64 and wave == copy_floor // CH and 4 * case.items > copy_floor
    else:
        assert copy_floor == 0
    if kind == 'capped':
        assert 4 * case.items < n // 64 and wave == 4 * case.items // CH
    elif kind != 'large' and not case.chunk:
        assert wave == max(n // 64 // CH, 1) and n // 64 < 4 * case.items
    if kind == 'long':
        a, b = sorted(LONG_USERS)
        assert all(deg[u] == k > wave * CH for u, k in LONG_USERS.items()) and b == a + 2 and deg[a + 1] == 0
        # they start in the last chunk of a wave: with every boundary one chunk early they run a wave later, so the
        # bound on these cases pins the wave of the users that run on through many
        assert all(rowptr[u] % (wave * CH) >= (wave - 1) * CH for u in LONG_USERS)
    if kind == 'sparse':
        assert n < case.users
    if case.chunk:
        assert len(launches) > 3 and max(b - a for a, b in launches) < case.users
    if case.degrees[0] == 'tails':
        lpr = row_lpr(case.d // 4)
        assert set(deg.tolist()) == set(range(2 * lpr + 2))
        assert all((deg == k).sum() >= 32 for k in (1, 2, 3, 4, 5, lpr, lpr + 1))


@pytest.mark.parametrize('case', CASES, ids=lambda c: c.name)
def test_case_rejection_sets_are_a_strict_superset(case):
    from qrec_b200 import engine as E
    c = case_data(case, E)
    rowptr, rrp, rc = c['rowptr'], c['rated_rowptr'], c['rated_cols']
    assert np.array_equal(rowptr, case_rowptr(case)) and len(c['i']) == len(c['u']) == rowptr[-1]
    assert c['i'].dtype == np.int32 and rc.dtype == np.int32 and rrp.dtype == np.int64
    rated = np.zeros((case.users if case.users <= 30_000 else 0, case.items if case.items <= 3_000 else 0), bool)
    if rated.size:                                   # every positive is in its user's rejection row
        rated[np.repeat(np.arange(case.users), np.diff(rrp)), rc] = True
        assert rated[c['u'], c['i']].all()
    extra = (rrp[-1] - len(np.unique(c['u'].astype(np.int64) * case.items + c['i']))) / rrp[-1]
    assert 0.25 < extra < 0.45, extra                # about a third of the ratings are under the threshold
    assert all(np.all(np.diff(rc[rrp[u]:rrp[u + 1]]) > 0) for u in range(0, case.users, 97))
    if case.degrees[0] == 'long':
        assert rrp[SATURATED_USER + 1] - rrp[SATURATED_USER] == case.items
        assert all(rrp[u + 1] - rrp[u] == 30 for u in LONG_USERS)
