"""The lane-group shape of libqrec's row-parallel launchers (qrec_b200/csrc/lane_shape.h), compiled for the host through
tests/host_shims/lane_shape_host.cpp.  A row of d floats is nvec = d / 4 float4s; one lane group of LPR lanes owns it,
VPL float4s per lane, and the throughput triple kernels keep UNROLL triples in flight per group.  Launchers capped at
d = 128 have no two-slice shape.  The warp-per-triple parity kernels take E = ceil(d / 32) elements per lane, rounded up
to a power of two."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('shim') / 'liblane_shape_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-Wall', '-Werror', '-fPIC', '-shared', '-I',
                           os.path.join(ROOT, 'qrec_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'host_shims', 'lane_shape_host.cpp'), '-o', out])
    L = C.CDLL(out)
    L.row_shape_host.restype = C.c_int
    L.row_shape_host.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.row_lpr_host.restype = C.c_int
    L.row_lpr_host.argtypes = [C.c_int]
    L.lane_elems_host.restype = C.c_int
    L.lane_elems_host.argtypes = [C.c_int]
    return L


def shape(lib, nvec, max_d):
    out = (C.c_int * 3)()
    assert lib.row_shape_host(nvec, max_d, out) == 0
    return tuple(out)


# (largest nvec, (LPR, VPL, UNROLL)) in increasing nvec
WIDE_TABLE = [(4, (4, 1, 2)), (8, (8, 1, 4)), (16, (16, 1, 4)), (32, (32, 1, 4)), (64, (32, 2, 2))]


def expected(nvec, table):
    return next(s for top, s in table if nvec <= top)


def test_row_shape_up_to_d256(lib):
    got = {nvec: shape(lib, nvec, 256) for nvec in range(1, 65)}
    assert got == {nvec: expected(nvec, WIDE_TABLE) for nvec in range(1, 65)}


def test_row_shape_up_to_d128_has_no_two_slice_shape(lib):
    got = {nvec: shape(lib, nvec, 128) for nvec in range(1, 65)}
    narrow = WIDE_TABLE[:-1]
    assert {nvec: got[nvec] for nvec in range(1, 33)} == {nvec: expected(nvec, narrow) for nvec in range(1, 33)}
    # d <= 128 is checked before the dispatch; past it the widest one-slice shape stands
    assert all(got[nvec] == (32, 1, 4) for nvec in range(33, 65))


def test_row_lpr_is_the_shape_lpr(lib):
    for nvec in range(1, 65):
        assert lib.row_lpr_host(nvec) == shape(lib, nvec, 256)[0] == shape(lib, nvec, 128)[0]


def test_lane_elems(lib):
    got = {d: lib.lane_elems_host(d) for d in range(1, 257)}
    assert got == {d: 1 if d <= 32 else 2 if d <= 64 else 4 if d <= 128 else 8 for d in range(1, 257)}
