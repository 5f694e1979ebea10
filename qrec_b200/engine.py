"""Python face of libqrec.so: thin, typed wrappers over the C ABI (include/qrec.h).

Tables and index arrays on the device are torch CUDA tensors (torch is plumbing: allocation,
streams, torch.distributed); every compute call below goes through ctypes into the hand-written
sm_90a kernels.  There is no CPU path here: device entry points raise if a tensor is not on a
CUDA device.
"""
import contextlib
import ctypes as C
import math

import numpy as np

from ._lib import lib, check, MTState, QRecError  # noqa: F401  (QRecError re-exported)


def _i32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _i64p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def version():
    return lib.qrec_version().decode()


def launch_count():
    return int(lib.qrec_launch_count())


# =============================================================================================
# K0 (compat): CPython `random` clone + the reference samplers (host)
# =============================================================================================
class RatedCSR(object):
    """Per-user item sets of the id-mapped training matrix, in the two orders the reference uses.

    `pos_*`   : insertion order of trainSet_u[user] restricted to rating >= 1 -- the iteration
                order of BPR.trainModel (model/ranking/BPR.py:22-25, 31-33).
    `sorted_*`: every rated item of the user, ascending ids -- the rejection set
                (`item_j in self.PositiveSet[user]`, BPR.py:36; `neg_item in trainSet_u[user]`,
                base/deepRecommender.py:48).  Duplicate (user,item) lines collapse, as in the
                reference's dict-of-dicts (data/rating.py:55).
    """

    def __init__(self, num_users, num_items, u_ids, i_ids, ratings=None, positive_threshold=1.0):
        u_ids = np.ascontiguousarray(u_ids, dtype=np.int64)
        i_ids = np.ascontiguousarray(i_ids, dtype=np.int64)
        n = u_ids.shape[0]
        if i_ids.shape[0] != n:
            raise QRecError('RatedCSR: u_ids and i_ids differ in length')
        r = None
        if ratings is not None:
            r = np.ascontiguousarray(ratings, dtype=np.float64)
            if r.shape[0] != n:
                raise QRecError('RatedCSR: ratings and ids differ in length')
        self.num_users, self.num_items = int(num_users), int(num_items)
        # qrec_build_rated_csr (csrc/host_csr.cpp): counting sort by user + a small sort per user, threaded
        self.sorted_rowptr = np.zeros(self.num_users + 1, dtype=np.int64)
        self.pos_rowptr = np.zeros(self.num_users + 1, dtype=np.int64)
        sorted_cols, pos_cols, possorted_cols = (np.empty(n, dtype=np.int32) for _ in range(3))
        check(lib.qrec_build_rated_csr(n, _i64p(u_ids), _i64p(i_ids), r.ctypes.data_as(C.POINTER(C.c_double)) if r is not None else None,
                                       self.num_users, self.num_items, float(positive_threshold), _i64p(self.sorted_rowptr),
                                       _i32p(sorted_cols), _i64p(self.pos_rowptr), _i32p(pos_cols), _i32p(possorted_cols)),
              'qrec_build_rated_csr')
        n_rated, n_pos = int(self.sorted_rowptr[-1]), int(self.pos_rowptr[-1])
        self.sorted_cols = np.ascontiguousarray(sorted_cols[:n_rated])
        self.pos_cols = np.ascontiguousarray(pos_cols[:n_pos])
        # the positives again, ascending ids: BPR.trainModel rejects against PositiveSet only
        # (model/ranking/BPR.py:36); identical to sorted_* when every rating is >= threshold
        if n_pos == n_rated:
            self.possorted_rowptr, self.possorted_cols = self.sorted_rowptr, self.sorted_cols
        else:
            self.possorted_rowptr = self.pos_rowptr
            self.possorted_cols = np.ascontiguousarray(possorted_cols[:n_pos])

    @property
    def num_positives(self):
        return int(self.pos_rowptr[-1])


class MT19937(object):
    """Bit-exact clone of CPython's `random.Random` for the calls the reference makes."""

    def __init__(self, seed=None):
        self._st = MTState()
        if seed is not None:
            self.seed(seed)

    def seed(self, s):
        check(lib.qrec_mt_seed(C.byref(self._st), abs(int(s))), 'qrec_mt_seed')

    def setstate(self, state):
        """Accepts random.getstate() or a uint32[625] array (624 words + index)."""
        if isinstance(state, tuple):
            assert state[0] == 3
            state = state[1]
        a = np.ascontiguousarray(state, dtype=np.uint32)
        assert a.shape == (625,)
        check(lib.qrec_mt_set_state(C.byref(self._st), a.ctypes.data_as(C.POINTER(C.c_uint32))),
              'qrec_mt_set_state')

    def getstate_array(self):
        a = np.empty(625, dtype=np.uint32)
        check(lib.qrec_mt_get_state(C.byref(self._st), a.ctypes.data_as(C.POINTER(C.c_uint32))),
              'qrec_mt_get_state')
        return a

    def getstate(self):
        return (3, tuple(int(x) for x in self.getstate_array()), None)

    def random(self):
        return float(lib.qrec_mt_random(C.byref(self._st)))

    def randbelow(self, n):
        return int(lib.qrec_mt_randbelow(C.byref(self._st), int(n)))

    def getrandbits32(self):
        return int(lib.qrec_mt_next_u32(C.byref(self._st)))

    def shuffle(self, x):
        assert x.dtype == np.int32 and x.flags.c_contiguous
        check(lib.qrec_mt_shuffle_i32(C.byref(self._st), x.shape[0], _i32p(x)), 'qrec_mt_shuffle_i32')

    def shuffle_pairs(self, a, b):
        assert a.dtype == np.int32 and b.dtype == np.int32 and a.shape == b.shape
        assert a.flags.c_contiguous and b.flags.c_contiguous
        check(lib.qrec_mt_shuffle_pairs_i32(C.byref(self._st), a.shape[0], _i32p(a), _i32p(b)),
              'qrec_mt_shuffle_pairs_i32')

    def data_split(self, n, test_ratio):
        keep = np.empty(n, dtype=np.uint8)
        check(lib.qrec_mt_data_split(C.byref(self._st), n, float(test_ratio),
                                     keep.ctypes.data_as(C.POINTER(C.c_uint8))), 'qrec_mt_data_split')
        return keep.astype(bool)

    def sample_bpr_epoch(self, csr, out=None):
        """One epoch of model/ranking/BPR.py:31-38 -> (u, i, j) int32 arrays."""
        n = csr.num_positives
        if out is None:
            out = (np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32))
        u, i, j = out
        check(lib.qrec_sample_bpr_epoch(C.byref(self._st), csr.num_users, csr.num_items,
                                        _i64p(csr.pos_rowptr), _i32p(csr.pos_cols),
                                        _i64p(csr.possorted_rowptr), _i32p(csr.possorted_cols),
                                        _i32p(u), _i32p(i), _i32p(j)), 'qrec_sample_bpr_epoch')
        return u, i, j

    def sample_pairwise(self, csr, u, out=None):
        """Negatives for a batch of users: base/deepRecommender.py:44-50."""
        u = np.ascontiguousarray(u, dtype=np.int32)
        j = np.empty(u.shape[0], np.int32) if out is None else out
        check(lib.qrec_sample_pairwise(C.byref(self._st), u.shape[0], csr.num_items, _i32p(u),
                                       _i64p(csr.sorted_rowptr), _i32p(csr.sorted_cols), _i32p(j)),
              'qrec_sample_pairwise')
        return j

    def sample_tbpr_epoch(self, csr, order, joint, weak, strong):
        """One epoch of TBPR's preference chains (model/ranking/TBPR.py:131-160) for the users `order` (ids, in the
        order positiveSet lists them); joint / weak / strong: (rowptr int64 [U+1], items int32) pools in list order.
        -> (u, a, b) int32 steps and the number of steps per listed user (int64)."""
        order = np.ascontiguousarray(order, dtype=np.int32)
        cap = 4 * int((csr.pos_rowptr[order.astype(np.int64) + 1] - csr.pos_rowptr[order.astype(np.int64)]).sum()) if order.size else 0
        u, a, b = (np.empty(max(cap, 1), np.int32) for _ in range(3))
        per_user = np.zeros(max(order.shape[0], 1), np.int64)
        n = C.c_int64(0)
        arrs = [(np.ascontiguousarray(rp, dtype=np.int64), np.ascontiguousarray(items, dtype=np.int32))
                for rp, items in (joint, weak, strong)]               # kept alive until the call returns
        for rp, _ in arrs:
            if rp.shape[0] != csr.num_users + 1:
                raise QRecError('sample_tbpr_epoch: a pool rowptr has %d entries for %d users' % (rp.shape[0], csr.num_users))
        pools = [p for rp, items in arrs for p in (_i64p(rp), _i32p(items))]
        check(lib.qrec_sample_tbpr_epoch(C.byref(self._st), order.shape[0], _i32p(order), csr.num_items,
                                         _i64p(csr.pos_rowptr), _i32p(csr.pos_cols), _i64p(csr.possorted_rowptr),
                                         _i32p(csr.possorted_cols), *pools, _i32p(u), _i32p(a), _i32p(b),
                                         _i64p(per_user), C.byref(n)), 'qrec_sample_tbpr_epoch')
        del arrs
        k = int(n.value)
        return u[:k].copy(), a[:k].copy(), b[:k].copy(), per_user[:order.shape[0]].copy()

    def sample_sbpr_batch(self, csr, fp_rowptr, fp_items, fp_counts, fp_sorted, u):
        """Social item, its friend count and the negative for a batch of users: model/ranking/SBPR.py:84-100."""
        u = np.ascontiguousarray(u, dtype=np.int32)
        k, j, w = (np.empty(u.shape[0], np.int32) for _ in range(3))
        check(lib.qrec_sample_sbpr_batch(C.byref(self._st), u.shape[0], csr.num_items, _i32p(u),
                                         _i64p(csr.sorted_rowptr), _i32p(csr.sorted_cols), _i64p(fp_rowptr),
                                         _i32p(fp_items), _i32p(fp_counts), _i32p(fp_sorted), _i32p(k), _i32p(j), _i32p(w)),
              'qrec_sample_sbpr_batch')
        return k, j, w

    def sample_pointwise(self, csr, u, i):
        """1 positive + 4 negatives per interaction: base/deepRecommender.py:65-76."""
        u = np.ascontiguousarray(u, dtype=np.int32)
        i = np.ascontiguousarray(i, dtype=np.int32)
        n = u.shape[0]
        ou, oi, oy = (np.empty(5 * n, np.int32) for _ in range(3))
        check(lib.qrec_sample_pointwise(C.byref(self._st), n, csr.num_items, _i32p(u), _i32p(i),
                                        _i64p(csr.sorted_rowptr), _i32p(csr.sorted_cols),
                                        _i32p(ou), _i32p(oi), _i32p(oy)), 'qrec_sample_pointwise')
        return ou, oi, oy


def bpr_order_depth(u, i, j, num_users, num_items):
    """Number of levels of the sequential loop's dependency DAG (host, O(n))."""
    u = np.ascontiguousarray(u, dtype=np.int32)
    i = np.ascontiguousarray(i, dtype=np.int32)
    j = np.ascontiguousarray(j, dtype=np.int32)
    depth = int(lib.qrec_bpr_order_depth(u.shape[0], _i32p(u), _i32p(i), _i32p(j), int(num_users), int(num_items)))
    if depth < 0:
        raise QRecError('qrec_bpr_order_depth: id out of range')
    return depth


def bpr_order_prepare(u, i, j, num_users, num_items):
    """Row-version numbers for the dependency-ordered kernel (host, O(n))."""
    u = np.ascontiguousarray(u, dtype=np.int32)
    i = np.ascontiguousarray(i, dtype=np.int32)
    j = np.ascontiguousarray(j, dtype=np.int32)
    n = u.shape[0]
    wu, wi, wj = (np.empty(n, np.int32) for _ in range(3))
    check(lib.qrec_bpr_order_prepare(n, _i32p(u), _i32p(i), _i32p(j), int(num_users), int(num_items),
                                     _i32p(wu), _i32p(wi), _i32p(wj)), 'qrec_bpr_order_prepare')
    return wu, wi, wj


def mf_order_prepare(u, i, num_users, num_items):
    """Row-version numbers of a pointwise (u, i) stream for mf_sgd_ordered (host, O(n))."""
    u = np.ascontiguousarray(u, dtype=np.int32)
    i = np.ascontiguousarray(i, dtype=np.int32)
    n = u.shape[0]
    wu, wi = np.empty(n, np.int32), np.empty(n, np.int32)
    check(lib.qrec_mf_order_prepare(n, _i32p(u), _i32p(i), int(num_users), int(num_items), _i32p(wu), _i32p(wi)),
          'qrec_mf_order_prepare')
    return wu, wi


def mf_order_depth(u, i, num_users, num_items):
    """Longest dependency chain of a pointwise stream (host, O(n))."""
    u = np.ascontiguousarray(u, dtype=np.int32)
    i = np.ascontiguousarray(i, dtype=np.int32)
    depth = int(lib.qrec_mf_order_depth(u.shape[0], _i32p(u), _i32p(i), int(num_users), int(num_items)))
    if depth < 0:
        raise QRecError('qrec_mf_order_depth: id out of range')
    return depth


# =============================================================================================
# device entry points
# =============================================================================================
def _torch():
    import torch
    return torch


def _dev(t, dtype, name):
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise QRecError('%s must be a CUDA tensor (the engine has no CPU path)' % name)
    if t.dtype != dtype:
        raise QRecError('%s must be %s, got %s' % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise QRecError('%s must be contiguous' % name)
    return t.data_ptr()


def _stream():
    return _torch().cuda.current_stream().cuda_stream


def sample_neg_philox(u, sorted_rowptr, sorted_cols, num_items, seed, epoch, out=None):
    torch = _torch()
    n = u.shape[0]
    if out is None:
        out = torch.empty(n, dtype=torch.int32, device=u.device)
    check(lib.qrec_sample_neg_philox(n, int(num_items), _dev(u, torch.int32, 'u'),
                                     _dev(sorted_rowptr, torch.int64, 'sorted_rowptr'),
                                     _dev(sorted_cols, torch.int32, 'sorted_cols'),
                                     int(seed), int(epoch), _dev(out, torch.int32, 'out'), _stream()),
          'qrec_sample_neg_philox')
    return out


def bpr_sgd_ordered(P, Q, u, i, j, wu, wi, wj, lr, reg_u, reg_i, loss, n_warps=0):
    """Parity mode: sequential-equivalent BPR.optimization over the triples in array order.
    n_warps: pollers to launch (0 = fill the GPU); ~4x the DAG width (n / bpr_order_depth) is best."""
    torch = _torch()
    f64 = P.dtype == torch.float64
    dt = torch.float64 if f64 else torch.float32
    n = u.shape[0]
    d = P.shape[1]
    assert Q.shape[1] == d
    ver_p = torch.zeros(P.shape[0], dtype=torch.int32, device=P.device)
    ver_q = torch.zeros(Q.shape[0], dtype=torch.int32, device=P.device)
    ticket = torch.zeros(1, dtype=torch.int64, device=P.device)
    fn = lib.qrec_bpr_sgd_ordered_f64 if f64 else lib.qrec_bpr_sgd_ordered_f32
    check(fn(_dev(P, dt, 'P'), _dev(Q, dt, 'Q'), d, n, _dev(u, torch.int32, 'u'),
             _dev(i, torch.int32, 'i'), _dev(j, torch.int32, 'j'), _dev(wu, torch.int32, 'wu'),
             _dev(wi, torch.int32, 'wi'), _dev(wj, torch.int32, 'wj'), ver_p.data_ptr(),
             ver_q.data_ptr(), ticket.data_ptr(), float(lr), float(reg_u), float(reg_i),
             _dev(loss, torch.float64, 'loss'), int(n_warps), _stream()), 'qrec_bpr_sgd_ordered')
    return loss


def bpr_sgd_batch(P, Q, u, i, j, lr, reg_u, reg_i, loss, tma=False):
    """Throughput mode: fused gather-dot-sigmoid-update-scatter-add over device triples.
    tma=True (d=64 only) scatters through the bulk-copy engine instead of per-lane REDG."""
    torch = _torch()
    n = u.shape[0]
    d = P.shape[1]
    assert Q.shape[1] == d and i.shape[0] == n and j.shape[0] == n
    fn = lib.qrec_bpr_sgd_batch_tma_f32 if tma else lib.qrec_bpr_sgd_batch_f32
    check(fn(_dev(P, torch.float32, 'P'), _dev(Q, torch.float32, 'Q'), d, n,
                                     _dev(u, torch.int32, 'u'), _dev(i, torch.int32, 'i'),
                                     _dev(j, torch.int32, 'j'), float(lr), float(reg_u),
                                     float(reg_i), _dev(loss, torch.float64, 'loss'), _stream()),
          'qrec_bpr_sgd_batch_f32')
    return loss


def bpr_sgd_usermajor(P, Q, rowptr, i, j, lr, reg_u, reg_i, loss):
    """Throughput mode in the reference's user-major order: P[u] register-resident per user."""
    torch = _torch()
    n_users = rowptr.shape[0] - 1
    assert i.shape[0] == j.shape[0]
    check(lib.qrec_bpr_sgd_usermajor_f32(_dev(P, torch.float32, 'P'), _dev(Q, torch.float32, 'Q'), P.shape[1], n_users,
                                         int(i.shape[0]), Q.shape[0],
                                         _dev(rowptr, torch.int64, 'rowptr'), _dev(i, torch.int32, 'i'),
                                         _dev(j, torch.int32, 'j'), float(lr), float(reg_u), float(reg_i),
                                         _dev(loss, torch.float64, 'loss'), _stream()), 'qrec_bpr_sgd_usermajor_f32')
    return loss


def bpr_epoch_usermajor(P, Q, rowptr, i, rated_rowptr, rated_cols, num_items, seed, epoch, lr, reg_u, reg_i, loss,
                        j_out=None):
    """A whole user-major epoch with fused Philox negative sampling (one launch)."""
    torch = _torch()
    check(lib.qrec_bpr_epoch_usermajor_f32(_dev(P, torch.float32, 'P'), _dev(Q, torch.float32, 'Q'), P.shape[1],
                                           rowptr.shape[0] - 1, int(i.shape[0]), _dev(rowptr, torch.int64, 'rowptr'),
                                           _dev(i, torch.int32, 'i'), _dev(rated_rowptr, torch.int64, 'rated_rowptr'),
                                           _dev(rated_cols, torch.int32, 'rated_cols'), int(num_items), int(seed),
                                           int(epoch), _dev(j_out, torch.int32, 'j_out') if j_out is not None else None,
                                           float(lr), float(reg_u), float(reg_i), _dev(loss, torch.float64, 'loss'),
                                           _stream()), 'qrec_bpr_epoch_usermajor_f32')
    return loss


def rated_signature(rated_rowptr, rated_cols):
    """512-bit rated-set signature per user ([n_users, 16] int32 storage of uint32 words) for the
    pre-testing sampler of bpr_epoch_usermajor_sig; static per data set."""
    torch = _torch()
    n_users = rated_rowptr.shape[0] - 1
    sig = torch.empty(n_users, 16, dtype=torch.int32, device=rated_rowptr.device)
    check(lib.qrec_rated_signature_build(n_users, _dev(rated_rowptr, torch.int64, 'rated_rowptr'),
                                         _dev(rated_cols, torch.int32, 'rated_cols'), sig.data_ptr(), _stream()),
          'qrec_rated_signature_build')
    return sig


def bpr_epoch_usermajor_sig(P, Q, rowptr, i, rated_rowptr, rated_cols, rated_sig, num_items, seed, epoch, lr, reg_u,
                            reg_i, loss, j_out=None):
    """bpr_epoch_usermajor with the signature pre-test in the sampler (same negatives, same update)."""
    torch = _torch()
    if rated_sig.shape != (rated_rowptr.shape[0] - 1, 16):
        raise QRecError('rated_sig must be [n_users, 16] (rated_signature)')
    check(lib.qrec_bpr_epoch_usermajor_sig_f32(_dev(P, torch.float32, 'P'), _dev(Q, torch.float32, 'Q'), P.shape[1],
                                               rowptr.shape[0] - 1, int(i.shape[0]), _dev(rowptr, torch.int64, 'rowptr'),
                                               _dev(i, torch.int32, 'i'), _dev(rated_rowptr, torch.int64, 'rated_rowptr'),
                                               _dev(rated_cols, torch.int32, 'rated_cols'),
                                               _dev(rated_sig, torch.int32, 'rated_sig'), int(num_items), int(seed),
                                               int(epoch), _dev(j_out, torch.int32, 'j_out') if j_out is not None else None,
                                               float(lr), float(reg_u), float(reg_i), _dev(loss, torch.float64, 'loss'),
                                               _stream()), 'qrec_bpr_epoch_usermajor_sig_f32')
    return loss


def bpr_sgd_staged(P, u, pos_i, pos_j, R, D, lr, reg_u, reg_i, loss):
    """K1 against item rows staged in R (row-sharded Q); item deltas come back in D."""
    torch = _torch()
    check(lib.qrec_bpr_sgd_staged_f32(_dev(P, torch.float32, 'P'), P.shape[1], u.shape[0], _dev(u, torch.int32, 'u'),
                                      _dev(pos_i, torch.int32, 'pos_i'), _dev(pos_j, torch.int32, 'pos_j'),
                                      _dev(R, torch.float32, 'R'), _dev(D, torch.float32, 'D'), float(lr),
                                      float(reg_u), float(reg_i), _dev(loss, torch.float64, 'loss'), _stream()),
          'qrec_bpr_sgd_staged_f32')
    return loss


def ubench_row_ops(table, n_ops, mode, seed=1):
    """Roofline aid: n_ops random 256-byte row gathers (mode 0) / scatter-adds (1) / one of each (2) on
    table [rows, 64] fp32 with no arithmetic (csrc/microbench.cu).  Perturbs the table by ~1e-9 per op."""
    torch = _torch()
    if table.dim() != 2 or table.shape[1] != 64:
        raise QRecError('ubench_row_ops: table must be [rows, 64] fp32')
    sink = torch.zeros(1, dtype=torch.float32, device=table.device)
    check(lib.qrec_ubench_row_ops_f32(_dev(table, torch.float32, 'table'), table.shape[0], int(n_ops), int(mode),
                                      int(seed) & 0xffffffff, sink.data_ptr(), _stream()), 'qrec_ubench_row_ops_f32')


def table_delta(Q, B, D, S=None):
    """D = Q - B (and S = D): this rank's not-yet-exchanged item-row updates (csrc/table_sync.cu)."""
    torch = _torch()
    check(lib.qrec_table_delta_f32(_dev(Q, torch.float32, 'Q'), _dev(B, torch.float32, 'B'), _dev(D, torch.float32, 'D'),
                                   _dev(S, torch.float32, 'S') if S is not None else None, Q.numel(), _stream()),
          'qrec_table_delta_f32')


def table_merge(Q, B, D, S):
    """Q += S - D (float atomics, commutes with a running K1), B += S; S = sum over ranks of D."""
    torch = _torch()
    check(lib.qrec_table_merge_f32(_dev(Q, torch.float32, 'Q'), _dev(B, torch.float32, 'B'), _dev(D, torch.float32, 'D'),
                                   _dev(S, torch.float32, 'S'), Q.numel(), _stream()), 'qrec_table_merge_f32')


def _ptr_array(ptrs):
    import ctypes as C
    return (C.c_void_p * len(ptrs))(*[int(p) for p in ptrs])


def table_reduce_scatter_p2p(peer_D_ptrs, rank, S, n):
    """This rank's slice of S = sum over ranks of their D (P2P loads over NVLink; symmetric-memory pointers)."""
    torch = _torch()
    check(lib.qrec_table_reduce_scatter_p2p_f32(_ptr_array(peer_D_ptrs), len(peer_D_ptrs), int(rank),
                                                _dev(S, torch.float32, 'S'), int(n), _stream()),
          'qrec_table_reduce_scatter_p2p_f32')


def table_gather_merge_p2p(peer_S_ptrs, Q, B, D):
    """All-gather of the summed slices from their owners fused with the merge (Q += S - D; B += S)."""
    torch = _torch()
    check(lib.qrec_table_gather_merge_p2p_f32(_ptr_array(peer_S_ptrs), len(peer_S_ptrs), _dev(Q, torch.float32, 'Q'),
                                              _dev(B, torch.float32, 'B'), _dev(D, torch.float32, 'D'), Q.numel(), _stream()),
          'qrec_table_gather_merge_p2p_f32')


def score_topn(U, V, user_ids, rated_rowptr, rated_cols, N, rated_value=0.0, out_ids=None, out_scores=None, tensor_cores=None):
    """K8: the N best items of every listed user in one kernel (scores, rated -> rated_value, top-N; nothing
    materialised).  Returns (ids int32 [n, N], scores fp32 [n, N]), best first, ties by ascending item id.
    tensor_cores: True = the wgmma 3xTF32 kernel (csrc/topn_tc.cu; d <= 64, multiple of 4), False = the fp32 SIMT kernel
    (csrc/topn_kernels.cu), None = the tensor-core kernel where the width allows it, else the SIMT kernel."""
    torch = _torch()
    if tensor_cores is None:
        tensor_cores = U.shape[1] <= 64 and U.shape[1] % 4 == 0
    fn, name = (lib.qrec_score_topn_tc_f32, 'qrec_score_topn_tc_f32') if tensor_cores else (lib.qrec_score_topn_f32, 'qrec_score_topn_f32')
    n = int(user_ids.shape[0])
    if U.shape[1] != V.shape[1]:
        raise QRecError('score_topn: U and V must have the same width')
    if out_ids is None:
        out_ids = torch.empty(n, N, dtype=torch.int32, device=U.device)
    if out_scores is None:
        out_scores = torch.empty(n, N, dtype=torch.float32, device=U.device)
    check(fn(_dev(U, torch.float32, 'U'), _dev(V, torch.float32, 'V'), U.shape[1], V.shape[0],
             _dev(user_ids, torch.int32, 'user_ids'), n, _dev(rated_rowptr, torch.int64, 'rated_rowptr'),
             _dev(rated_cols, torch.int32, 'rated_cols'), float(rated_value), int(N),
             _dev(out_ids, torch.int32, 'out_ids'), _dev(out_scores, torch.float32, 'out_scores'), _stream()), name)
    return out_ids, out_scores


def adj_normalize(rowptr, cols, pair, pair_w, deg, vals):
    """deg = weighted row sums, vals = D^-1/2 A D^-1/2 entries (fp32, the reference's operand order)."""
    torch = _torch()
    check(lib.qrec_adj_normalize_f32(rowptr.shape[0] - 1, _dev(rowptr, torch.int64, 'rowptr'), _dev(cols, torch.int32, 'cols'),
                                     _dev(pair, torch.int32, 'pair') if pair is not None else None,
                                     _dev(pair_w, torch.float32, 'pair_w') if pair_w is not None else None,
                                     _dev(deg, torch.float32, 'deg'), _dev(vals, torch.float32, 'vals'), _stream()),
          'qrec_adj_normalize_f32')
    return vals


def edge_keep_philox(n_lines, drop_rate, seed, tag, epoch, device, out=None):
    torch = _torch()
    if out is None:
        out = torch.empty(n_lines, dtype=torch.uint8, device=device)
    check(lib.qrec_edge_keep_philox(int(n_lines), float(drop_rate), int(seed), int(tag), int(epoch), _dev(out, torch.uint8, 'keep'),
                                    _stream()), 'qrec_edge_keep_philox')
    return out


def adj_line_weights(line_pair, keep, pair_w):
    torch = _torch()
    check(lib.qrec_adj_line_weights_f32(line_pair.shape[0], _dev(line_pair, torch.int32, 'line_pair'),
                                        _dev(keep, torch.uint8, 'keep') if keep is not None else None, pair_w.shape[0],
                                        _dev(pair_w, torch.float32, 'pair_w'), _stream()), 'qrec_adj_line_weights_f32')
    return pair_w


def adj_subgraph(rowptr, cols, pair, pair_w):
    """CSR (rowptr, cols, vals) of the edges with pair_w > 0, re-normalised with the sub-graph's own degrees."""
    torch = _torch()
    n_rows = rowptr.shape[0] - 1
    dev = rowptr.device
    deg = torch.empty(n_rows, dtype=torch.float32, device=dev)
    new_rowptr = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
    scratch = torch.empty((n_rows + 1 + 1023) // 1024 + 1, dtype=torch.int64, device=dev)
    args = (_dev(rowptr, torch.int64, 'rowptr'), _dev(pair, torch.int32, 'pair'), _dev(pair_w, torch.float32, 'pair_w'))
    check(lib.qrec_adj_subgraph_count(n_rows, args[0], args[1], args[2], deg.data_ptr(), new_rowptr.data_ptr(), scratch.data_ptr(),
                                      _stream()), 'qrec_adj_subgraph_count')
    nnz = int(new_rowptr[-1].item())                          # the one host round trip: the size of the new arrays
    new_cols = torch.empty(nnz, dtype=torch.int32, device=dev)
    new_vals = torch.empty(nnz, dtype=torch.float32, device=dev)
    check(lib.qrec_adj_subgraph_fill_f32(n_rows, args[0], _dev(cols, torch.int32, 'cols'), args[1], args[2], deg.data_ptr(),
                                         new_rowptr.data_ptr(), new_cols.data_ptr(), new_vals.data_ptr(), _stream()),
          'qrec_adj_subgraph_fill_f32')
    return new_rowptr, new_cols, new_vals


def bucket_requests(ids, rows_per_rank, world, cap, count, send, pos, overflow):
    """K7: requests -> fixed-capacity per-owner buckets on the device (csrc/dense_kernels.cu)."""
    torch = _torch()
    check(lib.qrec_bucket_requests(_dev(ids, torch.int32, 'ids'), ids.shape[0], int(rows_per_rank), int(world), int(cap),
                                   _dev(count, torch.int32, 'count'), _dev(send, torch.int32, 'send'), _dev(pos, torch.int32, 'pos'),
                                   _dev(overflow, torch.int32, 'overflow'), _stream()), 'qrec_bucket_requests')


def gemv_t(A, v, out, alpha=1.0, beta=0.0):
    """out = beta*out + alpha * A^T v (v None: column sums of A); A [rows, cols] fp32 with unit column stride (a
    row slice of a workspace is fine), out [cols]."""
    torch = _torch()
    ptr, ld = _strided_rows(A, 'A')
    check(lib.qrec_gemv_t_f32(ptr, max(ld, A.shape[1]), A.shape[0], A.shape[1], _dev(v, torch.float32, 'v') if v is not None else None,
                              float(alpha), float(beta), _dev(out, torch.float32, 'out'), _stream()), 'qrec_gemv_t_f32')
    return out


def sumsq(x, out):
    torch = _torch()
    fn = lib.qrec_sumsq_f64 if x.dtype == torch.float64 else lib.qrec_sumsq_f32
    check(fn(_dev(x, x.dtype, 'x'), x.numel(), _dev(out, torch.float64, 'out'), _stream()), 'qrec_sumsq')
    return out


def table_snapshot(src, dst):
    """dst = src for contiguous fp32 tables of the same size (csrc/bpr_kernels.cu: the user-major epoch's per-wave copy
    of the item table)."""
    torch = _torch()
    if src.numel() != dst.numel():
        raise QRecError('table_snapshot: src has %d elements, dst %d' % (src.numel(), dst.numel()))
    check(lib.qrec_table_snapshot_f32(_dev(src, torch.float32, 'src'), _dev(dst, torch.float32, 'dst'), src.numel(),
                                      _stream()), 'qrec_table_snapshot_f32')
    return dst


class HostPipeline(object):
    """qrec_ctx: copy/compute pipeline for epochs whose triples live in host memory."""

    def __init__(self, device=0, chunk_triples=1 << 22):
        self._ctx = C.c_void_p()
        check(lib.qrec_ctx_create(int(device), int(chunk_triples), C.byref(self._ctx)), 'qrec_ctx_create')

    def set_rated_signature(self, sig):
        """sig: rated_signature(...) of ALL users ([n_users, 16] int32 CUDA) or None; kept alive by the pipeline."""
        torch = _torch()
        self._sig = sig
        check(lib.qrec_ctx_set_rated_signature(self._ctx, _dev(sig, torch.int32, 'rated_sig') if sig is not None else None),
              'qrec_ctx_set_rated_signature')

    def close(self):
        if self._ctx:
            check(lib.qrec_ctx_destroy(self._ctx), 'qrec_ctx_destroy')
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def bpr_epoch(self, P, Q, u, i, j, lr, reg_u, reg_i):
        """u,i,j: host int32 (numpy arrays or CPU torch tensors; pinned gives overlap)."""
        torch = _torch()

        def hp(a, name):
            if isinstance(a, np.ndarray):
                assert a.dtype == np.int32 and a.flags.c_contiguous, name
                return a.ctypes.data, a.shape[0]
            assert (not a.is_cuda) and a.dtype == torch.int32 and a.is_contiguous(), name
            return a.data_ptr(), a.shape[0]

        pu, n = hp(u, 'u')
        pi, ni = hp(i, 'i')
        pj, nj = hp(j, 'j')
        assert n == ni == nj
        torch.cuda.current_stream().synchronize()   # tables may have pending work on torch's stream
        loss = C.c_double(0.0)
        check(lib.qrec_bpr_epoch_host(self._ctx, _dev(P, torch.float32, 'P'), _dev(Q, torch.float32, 'Q'),
                                      P.shape[1], n, pu, pi, pj, float(lr), float(reg_u), float(reg_i),
                                      C.byref(loss)), 'qrec_bpr_epoch_host')
        return loss.value


def _host_ptr(a, dtype_np, dtype_t, name):
    torch = _torch()
    if isinstance(a, np.ndarray):
        assert a.dtype == dtype_np and a.flags.c_contiguous, name
        return a.ctypes.data, a.shape[0]
    assert (not a.is_cuda) and a.dtype == dtype_t and a.is_contiguous(), name
    return a.data_ptr(), a.shape[0]


def _bpr_epoch_usermajor_host(self, P, Q, rowptr, i, rated_rowptr, rated_cols, num_items, seed, epoch, lr, reg_u, reg_i):
    """HostPipeline method: user-major epoch with the positives (CSR: rowptr int64, i int32) in HOST
    memory (pinned gives overlap) and fused device-side negative sampling; returns sum(-ln s)."""
    torch = _torch()
    prp, nr = _host_ptr(rowptr, np.int64, torch.int64, 'rowptr')
    pi, _ = _host_ptr(i, np.int32, torch.int32, 'i')
    torch.cuda.current_stream().synchronize()
    loss = C.c_double(0.0)
    check(lib.qrec_bpr_epoch_usermajor_host(self._ctx, _dev(P, torch.float32, 'P'), _dev(Q, torch.float32, 'Q'), P.shape[1],
                                            nr - 1, prp, pi, _dev(rated_rowptr, torch.int64, 'rated_rowptr'),
                                            _dev(rated_cols, torch.int32, 'rated_cols'), int(num_items), int(seed),
                                            int(epoch), float(lr), float(reg_u), float(reg_i), C.byref(loss)),
          'qrec_bpr_epoch_usermajor_host')
    return loss.value


HostPipeline.bpr_epoch_usermajor = _bpr_epoch_usermajor_host


def spmm_csr(rowptr, cols, vals, X, Y, acc=None, acc_scale=0.0, rowsplit=False):
    """Y = A @ X (CSR fp32); optional fused acc += acc_scale * Y.  `rowsplit` selects the plain
    row-partitioned kernel instead of the nnz-balanced default."""
    torch = _torch()
    n_rows = rowptr.shape[0] - 1
    d = X.shape[1]
    fn = lib.qrec_spmm_csr_rowsplit_f32 if rowsplit else lib.qrec_spmm_csr_f32
    check(fn(n_rows, int(cols.shape[0]), _dev(rowptr, torch.int64, 'rowptr'), _dev(cols, torch.int32, 'cols'),
                                _dev(vals, torch.float32, 'vals'), _dev(X, torch.float32, 'X'),
                                _dev(Y, torch.float32, 'Y'), d,
                                _dev(acc, torch.float32, 'acc') if acc is not None else None,
                                float(acc_scale), _stream()), 'qrec_spmm_csr_f32')
    return Y


def spmm_csr_scatter_rows(rowptr, cols, vals, src_rows, X, Y, acc=None, acc_scale=0.0):
    """Y[dst] += a * X[src] over the edge lists (CSR rows) of the source rows `src_rows`, after
    zero-filling Y: Y = B^T X for the CSR matrix B = (rowptr, cols, vals) restricted to those rows.
    For the symmetric joint adjacency this is Y = A X with an X whose non-zero rows are `src_rows`."""
    torch = _torch()
    assert X.shape[0] == rowptr.shape[0] - 1, 'X has one row per CSR row (source node)'
    check(lib.qrec_spmm_csr_scatter_rows_f32(Y.shape[0], src_rows.shape[0], _dev(src_rows, torch.int32, 'src_rows'),
                                             _dev(rowptr, torch.int64, 'rowptr'), _dev(cols, torch.int32, 'cols'),
                                             _dev(vals, torch.float32, 'vals'), _dev(X, torch.float32, 'X'),
                                             _dev(Y, torch.float32, 'Y'), X.shape[1],
                                             _dev(acc, torch.float32, 'acc') if acc is not None else None,
                                             float(acc_scale), _stream()), 'qrec_spmm_csr_scatter_rows_f32')
    return Y


def bpr_partial_scores(U, V, u, i, j, reg, y_part, loss):
    """Column-block step, part 1: y_part[k] = U[u_k] . (V[i_k] - V[j_k]) over the LOCAL columns; local L2 part into loss."""
    torch = _torch()
    check(lib.qrec_bpr_partial_scores_f32(_dev(U, torch.float32, 'U'), _dev(V, torch.float32, 'V'), U.shape[1], u.shape[0],
                                          _dev(u, torch.int32, 'u'), _dev(i, torch.int32, 'i'), _dev(j, torch.int32, 'j'), float(reg),
                                          _dev(y_part, torch.float32, 'y_part'), _dev(loss, torch.float64, 'loss'), _stream()),
          'qrec_bpr_partial_scores_f32')
    return y_part


def bpr_grad_from_scores(U, V, u, i, j, y_full, eps, reg, log_weight, gU, gV, loss):
    """Column-block step, part 2: gradients of the local columns from the full scores (the ranks' partial scores summed)."""
    torch = _torch()
    check(lib.qrec_bpr_grad_from_scores_f32(_dev(U, torch.float32, 'U'), _dev(V, torch.float32, 'V'), U.shape[1], u.shape[0],
                                            _dev(u, torch.int32, 'u'), _dev(i, torch.int32, 'i'), _dev(j, torch.int32, 'j'),
                                            _dev(y_full, torch.float32, 'y_full'), float(eps), float(reg), float(log_weight),
                                            _dev(gU, torch.float32, 'gU'), _dev(gV, torch.float32, 'gV'),
                                            _dev(loss, torch.float64, 'loss'), _stream()), 'qrec_bpr_grad_from_scores_f32')
    return loss


def spmm_csr_rows(rowptr, cols, vals, rows, X, Y=None, compact=False, acc=None, acc_scale=0.0):
    """The rows `rows` (int32, -1 = padding) of the product (rowptr, cols, vals) @ X: written to Y (row k of a compact Y,
    row rows[k] otherwise; Y may be None) and / or accumulated as acc[rows[k]] += acc_scale * row (distinct rows)."""
    torch = _torch()
    assert Y is not None or acc is not None
    check(lib.qrec_spmm_csr_rows_f32(rows.shape[0], _dev(rows, torch.int32, 'rows'), _dev(rowptr, torch.int64, 'rowptr'),
                                     _dev(cols, torch.int32, 'cols'), _dev(vals, torch.float32, 'vals'),
                                     _dev(X, torch.float32, 'X'), _dev(Y, torch.float32, 'Y') if Y is not None else None,
                                     1 if compact else 0, X.shape[1],
                                     _dev(acc, torch.float32, 'acc') if acc is not None else None, float(acc_scale),
                                     _stream()), 'qrec_spmm_csr_rows_f32')
    return Y


def bpr_grad_scatter(U, V, u, i, j, eps, reg, gU, gV, loss):
    torch = _torch()
    check(lib.qrec_bpr_grad_scatter_f32(_dev(U, torch.float32, 'U'), _dev(V, torch.float32, 'V'),
                                        U.shape[1], u.shape[0], _dev(u, torch.int32, 'u'),
                                        _dev(i, torch.int32, 'i'), _dev(j, torch.int32, 'j'),
                                        float(eps), float(reg), _dev(gU, torch.float32, 'gU'),
                                        _dev(gV, torch.float32, 'gV'), _dev(loss, torch.float64, 'loss'),
                                        _stream()), 'qrec_bpr_grad_scatter_f32')
    return loss


def bpr_grad_scatter_scaled(U, V, u, i, j, y_scale, eps, reg, gU, gV, loss):
    """bpr_grad_scatter with the per-sample score scale of SBPR's first loss term (SBPR.py:110-113):
    -ln(sigmoid(y_scale[k] * y_k) + eps)."""
    torch = _torch()
    if y_scale.shape[0] != u.shape[0]:
        raise QRecError('bpr_grad_scatter_scaled: y_scale has %d entries for %d samples' % (y_scale.shape[0], u.shape[0]))
    check(lib.qrec_bpr_grad_scatter_scaled_f32(_dev(U, torch.float32, 'U'), _dev(V, torch.float32, 'V'),
                                               U.shape[1], u.shape[0], _dev(u, torch.int32, 'u'),
                                               _dev(i, torch.int32, 'i'), _dev(j, torch.int32, 'j'),
                                               _dev(y_scale, torch.float32, 'y_scale'),
                                               float(eps), float(reg), _dev(gU, torch.float32, 'gU'),
                                               _dev(gV, torch.float32, 'gV'), _dev(loss, torch.float64, 'loss'),
                                               _stream()), 'qrec_bpr_grad_scatter_scaled_f32')
    return loss


def adam_dense_tf1(var, m, v, g, lr, t, beta1=0.9, beta2=0.999, eps=1e-8):
    torch = _torch()
    check(lib.qrec_adam_dense_tf1_f32(_dev(var, torch.float32, 'var'), _dev(m, torch.float32, 'm'),
                                      _dev(v, torch.float32, 'v'), _dev(g, torch.float32, 'g'),
                                      var.numel(), float(lr), float(beta1), float(beta2), float(eps),
                                      int(t), _stream()), 'qrec_adam_dense_tf1_f32')
    return var


def adam_lr_t(lr, t, beta1=0.9, beta2=0.999):
    """lr * sqrt(1 - beta2^t) / (1 - beta1^t) with the roundings of qrec_adam_dense_tf1_f32 (fp32 powers)."""
    import numpy as np
    b1p = np.float32(float(np.float32(beta1)) ** float(t))        # (float)pow((double)beta1_f32, (double)t)
    b2p = np.float32(float(np.float32(beta2)) ** float(t))
    return float(np.float32(lr) * np.sqrt(np.float32(1.0) - b2p) / (np.float32(1.0) - b1p))


def adam_dense_tf1_devstep(var, m, v, g, lr_t_dev, beta1=0.9, beta2=0.999, eps=1e-8):
    """adam_dense_tf1 with the step factor in a 1-element fp32 CUDA tensor (filled from adam_lr_t before a replay)."""
    torch = _torch()
    check(lib.qrec_adam_dense_tf1_devstep_f32(_dev(var, torch.float32, 'var'), _dev(m, torch.float32, 'm'), _dev(v, torch.float32, 'v'),
                                              _dev(g, torch.float32, 'g'), var.numel(), _dev(lr_t_dev, torch.float32, 'lr_t'),
                                              float(beta1), float(beta2), float(eps), _stream()), 'qrec_adam_dense_tf1_devstep_f32')
    return var


def axpby(dst, a, b, alpha, beta):
    torch = _torch()
    check(lib.qrec_axpby_f32(_dev(dst, torch.float32, 'dst'), _dev(a, torch.float32, 'a'),
                             _dev(b, torch.float32, 'b'), float(alpha), float(beta), dst.numel(),
                             _stream()), 'qrec_axpby_f32')
    return dst


# ---------------------------------------------------------------------------------------------
# K6 / dense helpers (SimGCL, NGCF)
# ---------------------------------------------------------------------------------------------
def simgcl_perturb(Emb, eps, seed, tag, step, acc=None, acc_scale=0.0, d_valid=0, row_offset=0):
    """E += sign(E) * l2_normalize(U[0,1)^d) * eps (SimGCL.py:33-35); row_offset = global id of Emb's row 0 when
    Emb is a block of a row-sharded table (the noise is a function of the global row)."""
    torch = _torch()
    check(lib.qrec_simgcl_perturb_rows_f32(_dev(Emb, torch.float32, 'E'), Emb.shape[0], int(row_offset), Emb.shape[1],
                                           int(d_valid), float(eps), int(seed), int(tag), int(step),
                                           _dev(acc, torch.float32, 'acc') if acc is not None else None,
                                           float(acc_scale), _stream()), 'qrec_simgcl_perturb_rows_f32')
    return Emb


def simgcl_perturb_listed(Ec, rows, eps, seed, tag, step, acc=None, acc_scale=0.0, d_valid=0, row_offset=0):
    """simgcl_perturb for a compact block: row k of Ec stands for table row rows[k] (-1 = padding, skipped);
    acc[rows[k]] += acc_scale * perturbed row."""
    torch = _torch()
    check(lib.qrec_simgcl_perturb_listed_f32(_dev(Ec, torch.float32, 'Ec'), _dev(rows, torch.int32, 'rows'), rows.shape[0],
                                             int(row_offset), Ec.shape[1], int(d_valid), float(eps), int(seed), int(tag),
                                             int(step), _dev(acc, torch.float32, 'acc') if acc is not None else None,
                                             float(acc_scale), _stream()), 'qrec_simgcl_perturb_listed_f32')
    return Ec


def gather_normalize(T, idx, Z, norms):
    torch = _torch()
    check(lib.qrec_gather_normalize_f32(_dev(T, torch.float32, 'T'), _dev(idx, torch.int32, 'idx'), idx.shape[0],
                                        T.shape[1], _dev(Z, torch.float32, 'Z'), _dev(norms, torch.float32, 'norms'),
                                        _stream()), 'qrec_gather_normalize_f32')
    return Z


def infonce_rows(S, tau, loss):
    torch = _torch()
    assert S.shape[0] == S.shape[1]
    check(lib.qrec_infonce_rows_f32(_dev(S, torch.float32, 'S'), S.shape[0], float(tau),
                                    _dev(loss, torch.float64, 'loss'), _stream()), 'qrec_infonce_rows_f32')
    return loss


def normalize_bwd_scatter(dZ, Z, norms, idx, scale, G):
    torch = _torch()
    check(lib.qrec_normalize_bwd_scatter_f32(_dev(dZ, torch.float32, 'dZ'), _dev(Z, torch.float32, 'Z'),
                                             _dev(norms, torch.float32, 'norms'), _dev(idx, torch.int32, 'idx'),
                                             idx.shape[0], Z.shape[1], float(scale), _dev(G, torch.float32, 'G'),
                                             _stream()), 'qrec_normalize_bwd_scatter_f32')
    return G


def sgemm(A, B, C, trans_a=False, trans_b=False, alpha=1.0, beta=0.0):
    """C = alpha * op(A) @ op(B) + beta * C for contiguous row-major fp32 matrices."""
    torch = _torch()
    M = A.shape[1] if trans_a else A.shape[0]
    K = A.shape[0] if trans_a else A.shape[1]
    N = B.shape[0] if trans_b else B.shape[1]
    assert (B.shape[1] if trans_b else B.shape[0]) == K and tuple(C.shape) == (M, N)
    check(lib.qrec_sgemm_f32(int(trans_a), int(trans_b), M, N, K, float(alpha), _dev(A, torch.float32, 'A'),
                             A.shape[1], _dev(B, torch.float32, 'B'), B.shape[1], float(beta),
                             _dev(C, torch.float32, 'C'), C.shape[1], _stream()), 'qrec_sgemm_f32')
    return C


def _strided_rows(t, name):
    """[rows, d] fp32 view whose rows are contiguous but may sit ld apart (a column block)."""
    torch = _torch()
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1):
        raise QRecError('%s must be a 2-D fp32 CUDA tensor with unit column stride' % name)
    return t.data_ptr(), t.stride(0)


def ngcf_act_fwd(Z, keep, training, seed, tag, step, H, out, norms):
    torch = _torch()
    po, ldo = _strided_rows(out, 'out')
    check(lib.qrec_ngcf_act_fwd_f32(_dev(Z, torch.float32, 'Z'), Z.shape[0], Z.shape[1], float(keep), int(training),
                                    int(seed), int(tag), int(step), _dev(H, torch.float32, 'H'), po, ldo,
                                    _dev(norms, torch.float32, 'norms'), _stream()), 'qrec_ngcf_act_fwd_f32')


def ngcf_act_bwd(dOut, dH_extra, H, Z, norms, keep, training, seed, tag, step, dZ):
    torch = _torch()
    pd, ldd = _strided_rows(dOut, 'dOut')
    check(lib.qrec_ngcf_act_bwd_f32(pd, ldd,
                                    _dev(dH_extra, torch.float32, 'dH_extra') if dH_extra is not None else None,
                                    _dev(H, torch.float32, 'H'), _dev(Z, torch.float32, 'Z'),
                                    _dev(norms, torch.float32, 'norms'), Z.shape[0], Z.shape[1], float(keep),
                                    int(training), int(seed), int(tag), int(step), _dev(dZ, torch.float32, 'dZ'),
                                    _stream()), 'qrec_ngcf_act_bwd_f32')


def mul(dst, a, b):
    torch = _torch()
    check(lib.qrec_mul_f32(_dev(dst, torch.float32, 'dst'), _dev(a, torch.float32, 'a'), _dev(b, torch.float32, 'b'),
                           dst.numel(), _stream()), 'qrec_mul_f32')
    return dst


EPI_NONE, EPI_BIAS_RELU, EPI_RELU_MASK, EPI_BIAS = 0, 1, 2, 3


def _ld(t):
    """Leading dimension of a row-major 2-D tensor; torch reports stride 1 for a single-row view."""
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def tc_gemm(A, B, C, b_is_nk=False, epilogue=EPI_NONE, bias=None, mask=None):
    """C = epilogue(A @ B) (b_is_nk=False, B [K,N]) or epilogue(A @ B.T) (b_is_nk=True, B [N,K]) on the
    wgmma TF32 tensor-core path."""
    torch = _torch()
    M, K = A.shape
    N = B.shape[0] if b_is_nk else B.shape[1]
    assert (B.shape[1] if b_is_nk else B.shape[0]) == K and tuple(C.shape) == (M, N)
    check(lib.qrec_tc_gemm_tf32(int(b_is_nk), M, N, K, _dev(A, torch.float32, 'A'), _ld(A),
                                _dev(B, torch.float32, 'B'), _ld(B), _dev(C, torch.float32, 'C'), _ld(C),
                                int(epilogue), _dev(bias, torch.float32, 'bias') if bias is not None else None,
                                _dev(mask, torch.float32, 'mask') if mask is not None else None,
                                _ld(mask) if mask is not None else 0, _stream()), 'qrec_tc_gemm_tf32')
    return C


def tc_gemm_v2(A, B, C, b_is_nk=False, epilogue=EPI_NONE, bias=None, mask=None):
    """tc_gemm through the persistent TMA-fed pipeline (K <= 320; A taken as raw fp32 bits = TF32
    truncation).  1.4-1.7 x the v1 kernel at M = 327 680, slower below M ~ 50 000 (persistent pipeline start-up)."""
    torch = _torch()
    M, K = A.shape
    N = B.shape[0] if b_is_nk else B.shape[1]
    assert (B.shape[1] if b_is_nk else B.shape[0]) == K and tuple(C.shape) == (M, N)
    check(lib.qrec_tc_gemm_tf32_v2(int(b_is_nk), M, N, K, _dev(A, torch.float32, 'A'), _ld(A),
                                   _dev(B, torch.float32, 'B'), _ld(B), _dev(C, torch.float32, 'C'), _ld(C),
                                   int(epilogue), _dev(bias, torch.float32, 'bias') if bias is not None else None,
                                   _dev(mask, torch.float32, 'mask') if mask is not None else None,
                                   _ld(mask) if mask is not None else 0, _stream()), 'qrec_tc_gemm_tf32_v2')
    return C


def gather_rows(T, idx, out):
    """out[b, :d] = T[idx[b]]; `out` may be a column block of a wider matrix."""
    torch = _torch()
    po, ldo = _strided_rows(out, 'out')
    check(lib.qrec_gather_rows_f32(_dev(T, torch.float32, 'T'), _dev(idx, torch.int32, 'idx'), idx.shape[0],
                                   T.shape[1], po, ldo, _stream()), 'qrec_gather_rows_f32')
    return out


def scatter_add_rows(G, idx, src, scale=1.0):
    torch = _torch()
    ps, lds = _strided_rows(src, 'src')
    check(lib.qrec_scatter_add_rows_f32(_dev(G, torch.float32, 'G'), _dev(idx, torch.int32, 'idx'), idx.shape[0],
                                        G.shape[1], ps, lds, float(scale), _stream()), 'qrec_scatter_add_rows_f32')
    return G


def neumf_head(mode, training, UG, IG, H3, h_mf, h_mlp, r, reg, loss, y, dz, GMF, dUG, dIG, dH3):
    torch = _torch()
    f = lambda t, n: _dev(t, torch.float32, n) if t is not None else None      # noqa: E731
    n = (UG if UG is not None else H3).shape[0]
    d = (UG if UG is not None else H3).shape[1]
    check(lib.qrec_neumf_head_f32(int(mode), int(training), f(UG, 'UG'), f(IG, 'IG'), f(H3, 'H3'), f(h_mf, 'h_mf'),
                                  f(h_mlp, 'h_mlp'), f(r, 'r'), n, d, float(reg),
                                  _dev(loss, torch.float64, 'loss') if loss is not None else None,
                                  f(y, 'y'), f(dz, 'dz'), f(GMF, 'GMF'), f(dUG, 'dUG'), f(dIG, 'dIG'), f(dH3, 'dH3'),
                                  _stream()), 'qrec_neumf_head_f32')


def mask_rated(scores, users, rowptr, cols, value=0.0):
    torch = _torch()
    check(lib.qrec_mask_rated_f32(_dev(scores, torch.float32, 'scores'), scores.shape[0], scores.stride(0),
                                  _dev(users, torch.int32, 'users'), _dev(rowptr, torch.int64, 'rowptr'),
                                  _dev(cols, torch.int32, 'cols'), float(value), _stream()), 'qrec_mask_rated_f32')
    return scores


# ---------------------------------------------------------------------------------------------
# K9: rating-prediction MF family (kind 0 BasicMF, 1 PMF, 2 SVD)
# ---------------------------------------------------------------------------------------------
MF_KINDS = {'BasicMF': 0, 'PMF': 1, 'SVD': 2}


def _opt(t, dtype, name):
    return _dev(t, dtype, name) if t is not None else None


def mf_sgd_ordered(kind, P, Q, u, i, r, wu, wi, lr, reg_u, reg_i, loss, Bu=None, Bi=None, reg_b=0.0,
                   global_mean=0.0, n_warps=0):
    """Parity mode: sequential-equivalent pass over the entries (u, i, r) in array order."""
    torch = _torch()
    f64 = P.dtype == torch.float64
    dt = torch.float64 if f64 else torch.float32
    d = P.shape[1]
    assert Q.shape[1] == d and u.shape[0] == i.shape[0] == r.shape[0]
    ver_p = torch.zeros(P.shape[0], dtype=torch.int32, device=P.device)
    ver_q = torch.zeros(Q.shape[0], dtype=torch.int32, device=P.device)
    ticket = torch.zeros(1, dtype=torch.int64, device=P.device)
    fn = lib.qrec_mf_sgd_ordered_f64 if f64 else lib.qrec_mf_sgd_ordered_f32
    check(fn(int(kind), _dev(P, dt, 'P'), _dev(Q, dt, 'Q'), d, u.shape[0], _dev(u, torch.int32, 'u'),
             _dev(i, torch.int32, 'i'), _dev(r, dt, 'r'), _dev(wu, torch.int32, 'wu'), _dev(wi, torch.int32, 'wi'),
             ver_p.data_ptr(), ver_q.data_ptr(), ticket.data_ptr(), float(lr), float(reg_u), float(reg_i),
             _opt(Bu, dt, 'Bu'), _opt(Bi, dt, 'Bi'), float(reg_b), float(global_mean),
             _dev(loss, torch.float64, 'loss'), int(n_warps), _stream()), 'qrec_mf_sgd_ordered')
    return loss


def mf_sgd_batch(kind, P, Q, u, i, r, lr, reg_u, reg_i, loss, Bu=None, Bi=None, reg_b=0.0, global_mean=0.0,
                 max_inflight=0):
    """Throughput mode: fused gather-dot-step-scatter-add over device entries (fp32, d % 4 == 0).
    max_inflight > 0 bounds the entries concurrently between read and reduction (grid sizing)."""
    torch = _torch()
    d = P.shape[1]
    assert Q.shape[1] == d and u.shape[0] == i.shape[0] == r.shape[0]
    f32 = torch.float32
    check(lib.qrec_mf_sgd_batch_f32(int(kind), _dev(P, f32, 'P'), _dev(Q, f32, 'Q'), d, u.shape[0],
                                    _dev(u, torch.int32, 'u'), _dev(i, torch.int32, 'i'), _dev(r, f32, 'r'),
                                    float(lr), float(reg_u), float(reg_i), _opt(Bu, f32, 'Bu'), _opt(Bi, f32, 'Bi'),
                                    float(reg_b), float(global_mean), _dev(loss, torch.float64, 'loss'),
                                    int(max_inflight), _stream()),
          'qrec_mf_sgd_batch_f32')
    return loss


def mf_predict_pairs(P, Q, u, i, Bu=None, Bi=None, global_mean=0.0, out=None):
    """out[k] = P[u[k]].Q[i[k]] (+ global_mean + Bi + Bu): predictForRating for known pairs."""
    torch = _torch()
    f64 = P.dtype == torch.float64
    dt = torch.float64 if f64 else torch.float32
    if out is None:
        out = torch.empty(u.shape[0], dtype=dt, device=P.device)
    fn = lib.qrec_mf_predict_pairs_f64 if f64 else lib.qrec_mf_predict_pairs_f32
    check(fn(_dev(P, dt, 'P'), _dev(Q, dt, 'Q'), P.shape[1], u.shape[0], _dev(u, torch.int32, 'u'),
             _dev(i, torch.int32, 'i'), _opt(Bu, dt, 'Bu'), _opt(Bi, dt, 'Bi'), float(global_mean),
             _dev(out, dt, 'out'), _stream()), 'qrec_mf_predict_pairs')
    return out


# =============================================================================================
# K10: WRMF (implicit-feedback ALS) -- Gram matrix and per-row normal-equation solve
# =============================================================================================
_ROWS_FAILED = 'row(s) with normal equations that are not positive definite were left unchanged'


@contextlib.contextmanager
def _failures(n_failed, device, message):
    """Yields the n_failed counter of one ALS-family launch: the caller's, or, when the caller gave none, a zeroed
    one that is read back after the launch; a count above 0 in it raises QRecError(message % count)."""
    own = n_failed is None
    if own:
        torch = _torch()
        n_failed = torch.zeros(1, dtype=torch.int32, device=device)
    yield n_failed
    if own:
        bad = int(n_failed.item())
        if bad:
            raise QRecError(message % bad)


def als_row_order(rowptr):
    """Rows by decreasing entry count (ties by id): the order als_solve_rows hands rows to its persistent grid,
    so that one long row does not become the tail.  rowptr: host int64 array."""
    lengths = np.diff(np.asarray(rowptr, dtype=np.int64))
    return np.argsort(-lengths, kind='stable').astype(np.int32)


def als_gram(Z, G=None, workspace=None):
    """G = Z^T Z as a float64 [d, d] CUDA tensor for a float32 / float64 table Z (bitwise reproducible).
    workspace: optional uint8 CUDA tensor of at least qrec_als_gram_workspace_bytes(n, d) bytes, reused across calls."""
    torch = _torch()
    n, d = Z.shape
    if Z.dtype not in (torch.float32, torch.float64):
        raise QRecError('Z must be float32 or float64, got %s' % Z.dtype)
    need = int(lib.qrec_als_gram_workspace_bytes(n, d))
    if need < 0:
        check(need, 'qrec_als_gram_workspace_bytes')
    if G is None:
        G = torch.empty(d, d, dtype=torch.float64, device=Z.device)
    if workspace is None:
        workspace = torch.empty(max(need, 1), dtype=torch.uint8, device=Z.device)
    fn = lib.qrec_als_gram_f64 if Z.dtype == torch.float64 else lib.qrec_als_gram_f32
    check(fn(_dev(Z, Z.dtype, 'Z'), n, d, _dev(G, torch.float64, 'G'), _dev(workspace, torch.uint8, 'workspace'),
             workspace.numel(), _stream()), 'qrec_als_gram')
    return G


def als_solve_rows(X, Z, G, rowptr, cols, vals, lam, alpha, row_order, loss=None, n_failed=None):
    """Solves the rows `row_order` of X against Z (WRMF.py:22-42 / 44-61): X[r] = (G + lam*I + alpha*sum v z z^T)^-1
    sum (1 + alpha*v) z over row r's entries (cols, vals) of the CSR (rowptr int64, cols int32, vals like X).
    loss: optional float64 CUDA tensor that accumulates sum (1 - x_old.z)^2.  n_failed: optional int32 CUDA tensor
    counting rows whose normal equations were not positive definite (left unchanged); when it is not given, the count
    is read back here and a failed row raises QRecError."""
    torch = _torch()
    d = X.shape[1]
    if X.dtype not in (torch.float32, torch.float64):
        raise QRecError('X must be float32 or float64, got %s' % X.dtype)
    dt = X.dtype
    if Z.shape[1] != d:
        raise QRecError('X and Z differ in width (%d, %d)' % (d, Z.shape[1]))
    fn = lib.qrec_als_solve_rows_f64 if dt == torch.float64 else lib.qrec_als_solve_rows_f32
    with _failures(n_failed, X.device, 'als_solve_rows: %d ' + _ROWS_FAILED) as n_failed:
        check(fn(_dev(X, dt, 'X'), _dev(Z, dt, 'Z'), _dev(G, torch.float64, 'G'), d, row_order.shape[0],
                 _dev(row_order, torch.int32, 'row_order'), _dev(rowptr, torch.int64, 'rowptr'),
                 _dev(cols, torch.int32, 'cols'), _dev(vals, dt, 'vals'), float(lam), float(alpha),
                 _opt(loss, torch.float64, 'loss'), _dev(n_failed, torch.int32, 'n_failed'), _stream()),
              'qrec_als_solve_rows')
    return X


# =============================================================================================
# K12: CoFactor -- SPPMI co-occurrence counts and the in-order item sweep
# =============================================================================================
def cooc_count(item_rowptr, item_users, num_users, filt):
    """Co-occurrence counts of CoFactor's SPPMI (CoFactor.py, initModel) on the device.  item_rowptr (int64
    [num_items + 1]) / item_users (int32): every item's DISTINCT users (Rating.rating_csr('item')).  Items with at
    least `filt` users are eligible; for eligible i != j the count of common users is kept when > filt.
    Returns the CSR (rowptr int64, cols int32 ascending per row, counts int32), symmetric."""
    torch = _torch()
    n_items = item_rowptr.shape[0] - 1
    _dev(item_rowptr, torch.int64, 'item_rowptr')
    _dev(item_users, torch.int32, 'item_users')
    dev = item_rowptr.device
    nnz = item_users.shape[0]
    if nnz == 0:                                  # no ratings: no pairs
        return (torch.zeros(n_items + 1, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int32, device=dev),
                torch.empty(0, dtype=torch.int32, device=dev))
    if int(item_users.min()) < 0 or int(item_users.max()) >= num_users:
        raise QRecError('cooc_count: a user id is outside [0, %d)' % num_users)
    deg = item_rowptr[1:] - item_rowptr[:-1]
    item_of = torch.repeat_interleave(torch.arange(n_items, dtype=torch.int32, device=dev), deg, output_size=nnz)
    # user-major transpose with ascending items: the item-major entries are in item order, the sort is stable
    user_items = item_of[torch.sort(item_users, stable=True).indices].contiguous()
    udeg = torch.bincount(item_users, minlength=num_users)
    user_rowptr = torch.zeros(num_users + 1, dtype=torch.int64, device=dev)
    torch.cumsum(udeg, 0, out=user_rowptr[1:])
    # eligible rows, the most user-item steps first (sum over the row's users of their degrees)
    work = torch.zeros(n_items, dtype=torch.int64, device=dev).index_add_(0, item_of.long(), udeg[item_users.long()])
    elig = torch.nonzero(deg >= filt).flatten()
    order = elig[torch.argsort(work[elig], descending=True, stable=True)].to(torch.int32).contiguous()
    row_nnz = torch.zeros(n_items, dtype=torch.int64, device=dev)
    args = (n_items, item_rowptr.data_ptr(), item_users.data_ptr(), user_rowptr.data_ptr(), user_items.data_ptr(),
            order.shape[0], order.data_ptr(), int(filt))
    check(lib.qrec_cooc_count(*args, None, row_nnz.data_ptr(), None, None, _stream()), 'qrec_cooc_count')
    rowptr = torch.zeros(n_items + 1, dtype=torch.int64, device=dev)
    torch.cumsum(row_nnz, 0, out=rowptr[1:])
    total = int(rowptr[-1])
    cols = torch.empty(total, dtype=torch.int32, device=dev)
    counts = torch.empty(total, dtype=torch.int32, device=dev)
    if total:
        check(lib.qrec_cooc_count(*args, rowptr.data_ptr(), None, cols.data_ptr(), counts.data_ptr(), _stream()),
              'qrec_cooc_count')
    return rowptr, cols, counts


def sppmi_csr(item_rowptr, item_users, num_users, k, filt, dtype=None):
    """CoFactor's SPPMI matrix (CoFactor.py, initModel) as a device CSR (rowptr int64, cols int32 ascending, vals):
    with f_i the sum of row i's kept counts and D the sum of all f, the value of a pair is
    max(log((count*D) / (f_i*f_j)) - log(k), 0) in float64, kept when > 0, then divided by the largest value.
    k < 1 counts as 1.  vals are float64, or `dtype`."""
    torch = _torch()
    rowptr, cols, counts = cooc_count(item_rowptr, item_users, num_users, filt)
    n_items = rowptr.shape[0] - 1
    dev = rowptr.device
    rows = torch.repeat_interleave(torch.arange(n_items, device=dev), rowptr[1:] - rowptr[:-1], output_size=cols.shape[0])
    cnt = counts.to(torch.float64)
    f = torch.zeros(n_items, dtype=torch.float64, device=dev).index_add_(0, rows, cnt)   # integer sums: exact
    D = f.sum()
    val = torch.log((cnt * D) / (f[rows] * f[cols.long()])) - math.log(max(int(k), 1))
    keep = val > 0
    val, cols, rows = val[keep], cols[keep].contiguous(), rows[keep]
    out_rowptr = torch.zeros(n_items + 1, dtype=torch.int64, device=dev)
    torch.cumsum(torch.bincount(rows, minlength=n_items), 0, out=out_rowptr[1:])
    if val.numel():
        val = val / val.max()
    return out_rowptr, cols, val.to(dtype or torch.float64).contiguous()


def cofactor_item_sweep(Y, G, w, c, X, XtX, item_csr, sppmi, lam, gamma, alpha, n_failed=None, stamps=None,
                        sweep=1):
    """One in-order item half-epoch of CoFactor (CoFactor.py, trainModel, item loop) on the device, in place on Y, G
    (float32 / float64 [num_items, d]) and w, c ([num_items], like Y); X ([num_users, d], like Y) is only read and
    XtX = X^T X is float64 (als_gram).  item_csr: (rowptr int64, users int32, ratings like Y), rating_csr('item');
    sppmi: (rowptr int64, cols int32, vals like Y), symmetric (sppmi_csr).  lam regularises Y, gamma G, alpha is the
    confidence scale.  Contexts c < i are read after their own update, c > i before it, as in the sequential loop.
    stamps (int32 [num_items], all sweep - 1) lets a caller reuse one stamp array across sweeps 1, 2, ...; without
    it a zeroed array is used for sweep 1.  n_failed: optional int32 CUDA tensor counting systems that were not
    positive definite (their rows left unchanged); when it is not given, the count is read back here and a failed
    system raises QRecError."""
    torch = _torch()
    dt = Y.dtype
    if dt not in (torch.float32, torch.float64):
        raise QRecError('Y must be float32 or float64, got %s' % dt)
    n_items, d = Y.shape
    if G.shape != Y.shape or X.dim() != 2 or X.shape[1] != d:
        raise QRecError('cofactor_item_sweep: G must have the shape of Y and X its width')
    if w.shape != (n_items,) or c.shape != (n_items,):
        raise QRecError('cofactor_item_sweep: w and c need one entry per item')
    if tuple(XtX.shape) != (d, d):
        raise QRecError('cofactor_item_sweep: XtX must be [%d, %d]' % (d, d))
    irp, icol, ival = item_csr
    srp, scol, sval = sppmi
    if irp.shape[0] != n_items + 1 or srp.shape[0] != n_items + 1:
        raise QRecError('cofactor_item_sweep: item and SPPMI rowptrs need %d entries' % (n_items + 1))
    if icol.shape[0] != ival.shape[0] or scol.shape[0] != sval.shape[0]:
        raise QRecError('cofactor_item_sweep: cols and vals differ in length')
    if stamps is None:
        stamps, sweep = torch.zeros(n_items, dtype=torch.int32, device=Y.device), 1
    elif stamps.shape != (n_items,) or (n_items and not bool((stamps == sweep - 1).all())):
        raise QRecError('cofactor_item_sweep: stamps must hold %d (sweep - 1) for every item' % (sweep - 1))
    ticket = torch.zeros(1, dtype=torch.int64, device=Y.device)
    fn = lib.qrec_cofactor_item_sweep_f64 if dt == torch.float64 else lib.qrec_cofactor_item_sweep_f32
    with _failures(n_failed, Y.device, 'cofactor_item_sweep: %d system(s) that are not positive definite left their '
                   'rows unchanged') as n_failed:
        check(fn(_dev(Y, dt, 'Y'), _dev(G, dt, 'G'), _dev(w, dt, 'w'), _dev(c, dt, 'c'), _dev(X, dt, 'X'),
                 _dev(XtX, torch.float64, 'XtX'), d, n_items, _dev(irp, torch.int64, 'item rowptr'),
                 _dev(icol, torch.int32, 'item users'), _dev(ival, dt, 'item ratings'),
                 _dev(srp, torch.int64, 'SPPMI rowptr'), _dev(scol, torch.int32, 'SPPMI cols'),
                 _dev(sval, dt, 'SPPMI vals'), float(lam), float(gamma), float(alpha),
                 _dev(stamps, torch.int32, 'stamps'), int(sweep), ticket.data_ptr(),
                 _dev(n_failed, torch.int32, 'n_failed'), _stream()), 'qrec_cofactor_item_sweep')
    return Y


# =============================================================================================
# K13: ExpoMF -- exposure posterior and weighted normal equations, fused per row
# =============================================================================================
def _exposure_checks(name, X, Z, rowptr, cols, row_order):
    """The checks expomf_half_epoch and serec_half_epoch (`name`) share: X [n, d] and Z [m, d] float32 and not one
    table, 1 <= d <= 128, and a CSR of n rows into [0, m) with row_order a list of its rows.  Returns (n, d, m)."""
    f32 = _torch().float32
    for t, tname in ((X, 'X'), (Z, 'Z')):
        if t.dtype != f32:
            raise QRecError('%s: %s must be float32, got %s' % (name, tname, t.dtype))
    if X.dim() != 2 or Z.dim() != 2 or Z.shape[1] != X.shape[1]:
        raise QRecError('%s: X and Z must be 2-D tables of one width' % name)
    n, d = X.shape
    m = Z.shape[0]
    if not 1 <= d <= 128:
        raise QRecError('%s: d=%d unsupported (1..128)' % (name, d))
    if X.data_ptr() == Z.data_ptr():
        raise QRecError('%s: X and Z must be different tables' % name)
    if rowptr.shape != (n + 1,):
        raise QRecError('%s: rowptr needs %d entries' % (name, n + 1))
    if row_order.dim() != 1 or row_order.shape[0] > n:
        raise QRecError('%s: row_order must be a list of at most %d rows' % (name, n))
    if row_order.numel() and (int(row_order.min()) < 0 or int(row_order.max()) >= n):
        raise QRecError('%s: a row of row_order is outside [0, %d)' % (name, n))
    nnz = cols.shape[0]
    if int(rowptr[0]) != 0 or int(rowptr[-1]) != nnz or (n and bool((rowptr[1:] < rowptr[:-1]).any())):
        raise QRecError('%s: rowptr must rise from 0 to len(cols) = %d' % (name, nnz))
    if nnz and (int(cols.min()) < 0 or int(cols.max()) >= m):
        raise QRecError('%s: a column is outside [0, %d)' % (name, m))
    return n, d, m


def expomf_half_epoch(X, Z, rowptr, cols, mu, mu_by_row, lam, lam_y, row_order, mu_out=None, a=1.0, b=99.0,
                      n_failed=None, max_ctas=0):
    """One ExpoMF half-epoch (ExpoMF.py: recompute_factors) in place on the rows `row_order` of X (float32 [n, d])
    against every row of Z (float32 [m, d]): with s = x_old.z and the exposure posterior
    A = (p + 1e-8) / (p + 1e-8 + (1 - mu) / mu), p = sqrt(lam_y/2/pi) exp(-lam_y s^2 / 2), set to 1 on row r's
    observed columns (rowptr int64 [n + 1], cols int32 < m),
        X[r] = (sum_k A_k z_k z_k^T + lam*I)^-1 sum_{observed k} z_k.
    mu (float32) is indexed by X's row when mu_by_row ([n]), else by Z's row ([m]).  mu_out (float32 [n], item half):
    also writes mu_out[r] = (a + sum_k A_k - 1) / (a + b + m - 2) with A from the new X[r] and mu[r] (mu then needs
    n entries; mu_out must not be mu).  max_ctas > 0 caps the grid (the result does not depend on it).  n_failed:
    optional int32 CUDA tensor counting rows whose system was not positive definite (left unchanged); when it is not
    given, the count is read back here and a failed row raises QRecError."""
    torch = _torch()
    f32 = torch.float32
    n, d, m = _exposure_checks('expomf_half_epoch', X, Z, rowptr, cols, row_order)
    if mu.dtype != f32:
        raise QRecError('expomf_half_epoch: mu must be float32, got %s' % mu.dtype)
    want = n if mu_by_row else m
    if mu.shape != (want,):
        raise QRecError('expomf_half_epoch: mu indexed by %s needs %d entries, got %s'
                        % ('row' if mu_by_row else 'column', want, tuple(mu.shape)))
    if mu_out is not None:
        if mu_out.dtype != f32 or mu_out.shape != (n,) or mu.shape != (n,):
            raise QRecError('expomf_half_epoch: mu_out and mu need one float32 entry per row (%d)' % n)
        if mu_out.data_ptr() == mu.data_ptr():
            raise QRecError('expomf_half_epoch: mu_out must be a buffer of its own, not mu')
    with _failures(n_failed, X.device, 'expomf_half_epoch: %d ' + _ROWS_FAILED) as n_failed:
        check(lib.qrec_expomf_solve_rows_f32(_dev(X, f32, 'X'), _dev(Z, f32, 'Z'), d, m, row_order.shape[0],
                                             _dev(row_order, torch.int32, 'row_order'),
                                             _dev(rowptr, torch.int64, 'rowptr'), _dev(cols, torch.int32, 'cols'),
                                             _dev(mu, f32, 'mu'), int(bool(mu_by_row)), _opt(mu_out, f32, 'mu_out'),
                                             float(lam), float(lam_y), float(a), float(b), int(max_ctas),
                                             _dev(n_failed, torch.int32, 'n_failed'), _stream()),
              'qrec_expomf_solve_rows_f32')
    return X


# =============================================================================================
# K14: SERec -- ExpoMF's fused row solve with the social exposure prior evaluated per pair
# =============================================================================================
def serec_half_epoch(X, Z, rowptr, cols, asum, deg, row_is_user, lam, lam_y, row_order, asum_out=None, mu0=0.01,
                     a=1.0, b=99.0, s=2.2, n_failed=None, max_ctas=0):
    """One SERec half-epoch (SERec.py: recompute_factors) in place on the rows `row_order` of X (float32 [n, d])
    against every row of Z (float32 [m, d]), as expomf_half_epoch with the prior of each (user, item) pair
        mu(u, i) = (a + A_i + (s-1)*deg_u*A_i - 1) / (a + b + (s-1)*deg_u*A_i + U - 2)
    from asum (float64, A_i: each item's summed posterior) and deg (int32, each user's number of followees), or the
    uniform mu0 for every pair when asum is None.  row_is_user: X's rows are the users (asum [m], deg [n], U = n) or
    the items (asum [n], deg [m], U = m); the reference's item half takes the user branch when U == I.  asum_out
    (float64 [n], item half, a buffer of its own): also writes asum_out[r] = sum_k A_k with A from the new X[r] and
    mu(k, r), 1 on row r's observed columns -- asum then needs n entries and deg m.  max_ctas > 0 caps the grid (the
    result does not depend on it).  n_failed: optional int32 CUDA tensor counting rows whose system was not positive
    definite (left unchanged); when it is not given, the count is read back here and a failed row raises QRecError."""
    torch = _torch()
    f32, f64, i32 = torch.float32, torch.float64, torch.int32
    n, d, m = _exposure_checks('serec_half_epoch', X, Z, rowptr, cols, row_order)
    n_users, n_items = (n, m) if row_is_user else (m, n)
    if asum is not None and (asum.dtype != f64 or asum.shape != (n_items,)):
        raise QRecError('serec_half_epoch: asum needs one float64 entry per item (%d), got %s %s'
                        % (n_items, asum.dtype, tuple(asum.shape)))
    if deg.dtype != i32 or deg.shape != (n_users,):
        raise QRecError('serec_half_epoch: deg needs one int32 entry per user (%d), got %s %s'
                        % (n_users, deg.dtype, tuple(deg.shape)))
    if n_users and int(deg.min()) < 0:
        raise QRecError('serec_half_epoch: deg must not be negative')
    if asum_out is not None:
        if asum_out.dtype != f64 or asum_out.shape != (n,) or n != n_items:
            raise QRecError('serec_half_epoch: asum_out needs one float64 entry per row (%d), and the rows must be '
                            'the items' % n)
        if asum is not None and asum_out.data_ptr() == asum.data_ptr():
            raise QRecError('serec_half_epoch: asum_out must be a buffer of its own, not asum')
    with _failures(n_failed, X.device, 'serec_half_epoch: %d ' + _ROWS_FAILED) as n_failed:
        check(lib.qrec_serec_solve_rows_f32(_dev(X, f32, 'X'), _dev(Z, f32, 'Z'), d, m, row_order.shape[0],
                                            _dev(row_order, i32, 'row_order'), _dev(rowptr, torch.int64, 'rowptr'),
                                            _dev(cols, i32, 'cols'), _opt(asum, f64, 'asum'), float(mu0),
                                            _dev(deg, i32, 'deg'), int(bool(row_is_user)),
                                            _opt(asum_out, f64, 'asum_out'), float(lam), float(lam_y), float(a),
                                            float(b), float(s), n_users, int(max_ctas), _dev(n_failed, i32, 'n_failed'),
                                            _stream()),
              'qrec_serec_solve_rows_f32')
    return X


# =============================================================================================
# K11: SVD++ -- in-order parity epoch and user-major closed-form fast epoch
# =============================================================================================
def _svdpp_tables(P, Q, Y, Bu, Bi, dt):
    d = P.shape[1]
    if P.dim() != 2 or Q.dim() != 2 or Y.dim() != 2 or Q.shape[1] != d or Y.shape[1] != d:
        raise QRecError('svdpp: P, Q, Y must be 2-D tables of one width')
    if Y.shape[0] != Q.shape[0] or Bu.shape[0] != P.shape[0] or Bi.shape[0] != Q.shape[0]:
        raise QRecError('svdpp: Y / Bi need one row per item of Q, Bu one per user of P')
    return [_dev(t, dt, name) for t, name in ((P, 'P'), (Q, 'Q'), (Y, 'Y'), (Bu, 'Bu'), (Bi, 'Bi'))], d


def svdpp_sgd_ordered(P, Q, Y, Bu, Bi, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y, global_mean, loss):
    """Parity mode (SVDPlusPlus.py:30-61): the entries (u, i, r) one after another in array order on one CTA.
    rowptr (int64 [num_users + 1]) / cols (int32): every user's distinct items in insertion order
    (Rating.rating_csr('user')).  Tables float64 or float32 (all five alike, r likewise); loss: float64 [1], += sum e^2."""
    torch = _torch()
    dt = P.dtype
    if dt not in (torch.float32, torch.float64):
        raise QRecError('P must be float32 or float64, got %s' % dt)
    if not (u.shape[0] == i.shape[0] == r.shape[0]):
        raise QRecError('svdpp_sgd_ordered: u, i, r differ in length')
    if rowptr.shape[0] != P.shape[0] + 1:
        raise QRecError('svdpp_sgd_ordered: rowptr has %d entries for %d users' % (rowptr.shape[0], P.shape[0]))
    (pP, pQ, pY, pBu, pBi), d = _svdpp_tables(P, Q, Y, Bu, Bi, dt)
    fn = lib.qrec_svdpp_sgd_ordered_f64 if dt == torch.float64 else lib.qrec_svdpp_sgd_ordered_f32
    check(fn(pP, pQ, pY, pBu, pBi, d, u.shape[0], _dev(u, torch.int32, 'u'), _dev(i, torch.int32, 'i'), _dev(r, dt, 'r'),
             _dev(rowptr, torch.int64, 'rowptr'), _dev(cols, torch.int32, 'cols'), float(lr), float(reg_u), float(reg_i),
             float(reg_b), float(reg_y), float(global_mean), _dev(loss, torch.float64, 'loss'), _stream()),
          'qrec_svdpp_sgd_ordered')
    return loss


def svdpp_epoch_usermajor(P, Q, Y, Bu, Bi, rowptr, cols, vals, row_order, lr, reg_u, reg_i, reg_b, reg_y, global_mean,
                          loss, max_users_in_flight=0):
    """Throughput mode: one user-major epoch over the CSR (rowptr int64, cols int32, vals fp32: every user's distinct
    items and ratings), users in `row_order` (int32; als_row_order gives longest first), fp32 tables whose width is
    a multiple of 4 up to 128.  max_users_in_flight: 0 fills the GPU, k > 0 runs at most k users at a time."""
    torch = _torch()
    f32 = torch.float32
    if rowptr.shape[0] != P.shape[0] + 1:
        raise QRecError('svdpp_epoch_usermajor: rowptr has %d entries for %d users' % (rowptr.shape[0], P.shape[0]))
    if cols.shape[0] != vals.shape[0]:
        raise QRecError('svdpp_epoch_usermajor: cols and vals differ in length')
    (pP, pQ, pY, pBu, pBi), d = _svdpp_tables(P, Q, Y, Bu, Bi, f32)
    check(lib.qrec_svdpp_epoch_usermajor_f32(pP, pQ, pY, pBu, pBi, d, row_order.shape[0],
                                             _dev(row_order, torch.int32, 'row_order'), _dev(rowptr, torch.int64, 'rowptr'),
                                             _dev(cols, torch.int32, 'cols'), _dev(vals, f32, 'vals'), float(lr),
                                             float(reg_u), float(reg_i), float(reg_b), float(reg_y), float(global_mean),
                                             _dev(loss, torch.float64, 'loss'), int(max_users_in_flight), _stream()),
          'qrec_svdpp_epoch_usermajor_f32')
    return loss
