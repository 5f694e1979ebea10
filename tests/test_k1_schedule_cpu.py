"""The wave schedule of the fused user-major BPR epoch (qrec_b200/csrc/um_waves.cuh), compiled for the host through
tests/host_shims/um_waves_host.cpp.  launch_usermajor deals each wave's users [wave_user[w], wave_user[w + 1]) to the
lane groups; those must be exactly the users that the chunk rule assigns to wave w: the launch's triples are cut into
chunks of 32, a chunk takes the users whose first triple lies in it (the launch's first user starts at the launch's
first triple, its last user ends at its last), and wave w is chunks [w * wave, (w + 1) * wave)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH = 32


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'libum_waves_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-I', os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'um_waves_host.cpp'), '-o', out])
    L = C.CDLL(out)
    L.um_wave_chunks_host.restype = C.c_longlong
    L.um_wave_chunks_host.argtypes = [C.c_longlong, C.c_longlong, C.c_int]
    L.um_wave_table_host.restype = C.c_longlong
    L.um_wave_table_host.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_int, C.c_void_p,
                                     C.c_longlong]
    return L


def wave_chunks(n, num_items, d):
    """The wave length in chunks, as launch_usermajor has always sized it."""
    copy_bytes = 2 * num_items * d * 4
    copy_floor = 8 * copy_bytes // (24 * d + 12) if copy_bytes > (8 << 20) else 0
    wave_triples = min(max(n // 64, copy_floor), 4 * num_items)
    return max(wave_triples // CH, 1)


def chunk_rule_waves(rowptr, n, trip_off, wave):
    """The chunk rule: for every user with triples in the launch, the wave that processes it and the triples
    [lo, hi) (relative to trip_off) it is processed over; users with none get wave -1."""
    rel = rowptr.astype(np.int64) - trip_off
    n_users = len(rowptr) - 1
    nchunks = (n + CH - 1) // CH
    lo = np.arange(nchunks, dtype=np.int64) * CH
    hi = np.minimum(lo + CH, n)
    # user of triple t: the smallest r with rel[r + 1] > t
    uu = np.minimum(np.searchsorted(rel[1:], lo, side='right'), n_users - 1)
    cut = (lo > 0) & (rel[uu] < lo)                      # a user that started in an earlier chunk belongs to it
    lo = np.where(cut, rel[np.minimum(uu + 1, n_users)], lo)
    inner = hi < n
    ub = np.minimum(np.searchsorted(rel[1:], hi, side='right'), n_users - 1)
    ext = inner & (rel[ub] < hi)                         # a user that starts in this chunk is processed whole here
    hi = np.where(ext, np.minimum(rel[np.minimum(ub + 1, n_users)], n), hi)
    live = lo < hi
    ch_id, lo, hi = np.nonzero(live)[0], lo[live], hi[live]
    assert np.all(lo[1:] == hi[:-1]) and (len(lo) == 0 or (lo[0] == 0 and hi[-1] == n)), 'chunks do not tile the launch'
    s = np.clip(rel[:-1], 0, n)
    e = np.clip(rel[1:], 0, n)
    has = s < e
    k = np.searchsorted(lo, s[has], side='right') - 1    # the chunk holding the user's first triple
    assert np.all(hi[k] >= e[has]), 'a user is split between chunks'
    wave_of = np.full(n_users, -1, np.int64)
    wave_of[has] = ch_id[k] // wave
    return wave_of, s, e


def check(lib, rowptr, n, trip_off, num_items, d):
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
    n_users = len(rowptr) - 1
    wave = wave_chunks(n, num_items, d)
    assert lib.um_wave_chunks_host(n, num_items, d) == wave
    cap = (n + CH - 1) // CH + 2
    table = np.zeros(cap, np.int32)
    nwaves = lib.um_wave_table_host(rowptr.ctypes.data, n_users, n, trip_off, num_items, d, table.ctypes.data, cap)
    assert nwaves == -(-((n + CH - 1) // CH) // wave)
    table = table[:nwaves + 1].astype(np.int64)
    assert np.all(np.diff(table) >= 0) and 0 <= table[0] and table[-1] <= n_users
    wave_of, s, e = chunk_rule_waves(rowptr, n, trip_off, wave)
    # the kernel runs user u of wave w over [max(rowptr[u] - trip_off, 0), min(rowptr[u + 1] - trip_off, n))
    in_wave = np.searchsorted(table, np.arange(n_users), side='right') - 1
    in_wave[(np.arange(n_users) < table[0]) | (np.arange(n_users) >= table[-1])] = -1
    has = s < e
    np.testing.assert_array_equal(in_wave[has], wave_of[has])
    return nwaves, wave


def test_bench_shape(lib):
    users, deg, items = 1_000_000, 50, 100_000
    rowptr = np.arange(users + 1, dtype=np.int64) * deg
    nwaves, wave = check(lib, rowptr, users * deg, 0, items, 64)
    assert (nwaves, wave) == (125, 12_500)


@pytest.mark.parametrize('seed', [0, 1])
def test_ragged_degrees_with_empty_users(lib, seed):
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 121, 50_000)
    deg[:7] = 0; deg[-5:] = 0; deg[1000:1100] = 0                  # empty users at both ends and a run of them inside
    rowptr = np.zeros(len(deg) + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    nwaves, _ = check(lib, rowptr, int(rowptr[-1]), 0, 5_000, 64)
    assert nwaves >= 64                                             # small table: the 64-waves floor


def test_user_longer_than_a_wave(lib):
    deg = np.full(300, 3, np.int64)
    deg[17] = 5_000; deg[18] = 0; deg[19] = 1_000                  # each spans several waves of 4 x 40 triples
    rowptr = np.zeros(len(deg) + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    n = int(rowptr[-1])
    nwaves, wave = check(lib, rowptr, n, 0, 40, 16)
    assert wave * CH < 5_000


@pytest.mark.parametrize('d,num_items', [(64, 5_000), (32, 100_000), (128, 300)])
def test_host_pipeline_chunk_with_trip_off(lib, d, num_items):
    """One chunk of whole users of a larger epoch, as the host pipeline launches it: rowptr holds the global offsets
    of users [ua, ub], the launch's triples start at trip_off = rowptr[ua]."""
    rng = np.random.default_rng(d)
    deg = rng.integers(0, 90, 40_000)
    full = np.zeros(len(deg) + 1, np.int64); full[1:] = np.cumsum(deg)
    for ua, ub in ((0, 9_000), (9_000, 9_001), (12_345, 31_000), (31_000, 40_000)):
        rp = full[ua:ub + 1]
        n = int(rp[-1] - rp[0])
        if n:
            check(lib, rp, n, int(rp[0]), num_items, d)


def test_cut_launch_ends(lib):
    """A launch that starts and ends inside users: its first user starts at the launch's first triple, its last ends
    at its last."""
    rng = np.random.default_rng(7)
    deg = rng.integers(1, 200, 3_000)
    rowptr = np.zeros(len(deg) + 1, np.int64); rowptr[1:] = np.cumsum(deg)
    for trip_off, n in ((int(rowptr[5]) + 3, 100_000), (int(rowptr[0]) + 1, int(rowptr[-1]) - 2), (int(rowptr[40]), 777)):
        check(lib, rowptr, n, trip_off, 2_000, 64)
