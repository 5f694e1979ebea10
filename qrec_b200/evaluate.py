"""Batched top-N evaluation on the device (SURVEY.md 8f-1, "next" row).

The reference ranks one test user at a time: an I x d GEMV, rated items overwritten with 0, a
numba heap top-N (base/recommender.py:143-152).  Here blocks of users go through ONE kernel
(engine.score_topn, csrc/topn_kernels.cu / csrc/topn_tc.cu): score tile -> compare with the row's N-th best in
registers -> rated test for the survivors -> per-row candidate list; the [users x items] score matrix is never
written.  The kernel orders ties by ascending item id; the reference heap does not (it keeps a min-heap of
(score, id) and replaces its minimum only on a strictly larger score, so at a tie across the cut it keeps later
ids, and inside a tie it keeps heap order).  So the kernel is asked for N + 1 keys: a row whose N + 1 best scores
are all distinct has the heap's list already, and a row with equal scores among them is ranked again by
util.qmath.find_k_largest on its fp32 score row (engine.sgemm, rated items set to 0 by engine.mask_rated).  The
result is the reference heap's lists on the device's fp32 scores.  Opt-in through `engine=... -eval gpu`; the
default keeps the reference's host flow, whose float64 score strings are part of the recorded outputs.
"""
import numpy as np

from .util.qmath import find_k_largest

N_MAX = 100                  # base/recommender.py clamps -topN to <= 100; the kernels take N_MAX + 1 keys
RERANK_FLOATS = 1 << 26      # score floats of the tied rows ranked again at once (256 MB)


def batched_top_n(U, V, user_ids, csr, N, block=65536):
    """U [users,d], V [items,d]: fp32 CUDA tensors; user_ids: int array of rows of U to rank;
    csr: engine.RatedCSR of the training set; 1 <= N <= 100.  Returns (ids [n,N] int64, scores [n,N] float32),
    the lists of util.qmath.find_k_largest on the users' fp32 score rows with rated items scored 0."""
    import torch
    from . import engine as E
    if not 1 <= N <= N_MAX:
        raise ValueError('batched_top_n: N=%d must be in 1..%d' % (N, N_MAX))
    dev = U.device
    rowptr = torch.from_numpy(csr.sorted_rowptr).to(dev)
    cols = torch.from_numpy(csr.sorted_cols).to(dev)
    user_ids = np.ascontiguousarray(user_ids, dtype=np.int32)
    n, I = len(user_ids), V.shape[0]
    N = min(N, I)
    K = min(N + 1, I)                          # one key past the cut shows a tie across it
    out_ids = np.empty((n, N), np.int64)
    out_val = np.empty((n, N), np.float32)
    U, V = U.contiguous(), V.contiguous()
    for b in range(0, n, block):
        ub = torch.from_numpy(user_ids[b:b + block]).to(dev)
        ids, val = E.score_topn(U, V, ub, rowptr, cols, K, rated_value=0.0)
        ids, val = ids.cpu().numpy(), val.cpu().numpy()
        out_ids[b:b + ub.shape[0]] = ids[:, :N]
        out_val[b:b + ub.shape[0]] = val[:, :N]
        tied = np.nonzero((val[:, 1:] == val[:, :-1]).any(axis=1))[0]
        step = max(1, RERANK_FLOATS // I)
        for t in range(0, len(tied), step):
            rows = tied[t:t + step]
            users = torch.from_numpy(user_ids[b + rows]).to(dev)
            S = torch.empty(len(rows), I, dtype=torch.float32, device=dev)
            E.sgemm(U[users.long()].contiguous(), V, S, trans_b=True)
            E.mask_rated(S, users, rowptr, cols, 0.0)
            for r, s in zip(rows.tolist(), S.cpu().numpy()):
                out_ids[b + r], out_val[b + r] = find_k_largest(N, s)
    return out_ids, out_val
