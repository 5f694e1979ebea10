"""`GraphRecommender`: the adjacency builders of the graph models
(reference: base/graphRecommender.py:10-61).

`create_joint_sparse_adjaceny` returns the same scipy CSR (float32, D^-1/2 (R (+) R^T) D^-1/2 of
the (U+I)x(U+I) bipartite graph, duplicate interactions summed before normalisation);
`create_joint_sparse_adj_tensor` hands it to the device as a `DeviceCSR` (int64 rowptr, int32
cols, fp32 vals) -- the operand of the K2 SpMM kernel -- instead of building a tf.SparseTensor
from a Python list of (row, col) pairs.
"""
import numpy as np
import scipy.sparse as sp

from .deepRecommender import DeepRecommender


class DeviceCSR(object):
    """CSR operand resident in HBM; `matmul` is qrec_spmm_csr_f32."""

    def __init__(self, mat, device):
        import torch
        mat = mat.tocsr()
        mat.sort_indices()
        self._finish(mat.shape, torch.from_numpy(mat.indptr.astype(np.int64)).to(device),
                     torch.from_numpy(mat.indices.astype(np.int32)).to(device),
                     torch.from_numpy(mat.data.astype(np.float32)).to(device))
        self.split_row = None

    @classmethod
    def from_tensors(cls, shape, rowptr, cols, vals, split_row=None):
        """Wraps CSR arrays that already live on the device (graph_build.norm_adjacency_csr).  `split_row`: see
        set_split_row."""
        self = cls.__new__(cls)
        self._finish(tuple(shape), rowptr, cols, vals)
        self.set_split_row(split_row)
        return self

    def set_split_row(self, row):
        """The joint adjacency of a bipartite graph is two very different halves: `row` = num_users short user rows that
        gather item rows (a table that lives in the L2) and long item rows that gather user rows.  Lane groups working on
        50-entry and on 500-entry rows at the same time keep neither table's rows in the L2, so the halves are launched one
        after the other.  With a split row `matmul` issues the row-split
        kernel once per half; rows, arithmetic and results are those of the single launch."""
        n = self.shape[0]
        self.split_row = int(row) if (row is not None and 0 < int(row) < n) else None

    def _finish(self, shape, rowptr, cols, vals):
        self.shape = shape
        self.rowptr, self.cols, self.vals = rowptr, cols, vals
        self.nnz = int(cols.shape[0])
        # short, even rows: one lane group per row is fastest (no atomics); a long-tailed degree
        # distribution needs the nnz-balanced kernel or the hot rows serialise the launch
        lengths = rowptr[1:] - rowptr[:-1]
        self.rowsplit = bool(lengths.numel() == 0 or int(lengths.max().item()) <= 4096)

    def matmul_sparse_rows(self, X, src_rows, out, acc=None, acc_scale=0.0):
        """out = A @ X when only the rows `src_rows` of X are non-zero (A symmetric)."""
        from .. import engine
        return engine.spmm_csr_scatter_rows(self.rowptr, self.cols, self.vals, src_rows, X, out, acc=acc, acc_scale=acc_scale)

    def matmul_rows(self, X, rows, out=None, compact=False, acc=None, acc_scale=0.0):
        """The rows `rows` (int32, distinct, -1 = padding) of A @ X, stored into `out` and / or accumulated into acc."""
        from .. import engine
        return engine.spmm_csr_rows(self.rowptr, self.cols, self.vals, rows, X, out, compact=compact, acc=acc, acc_scale=acc_scale)

    def matmul(self, X, out, acc=None, acc_scale=0.0):
        from .. import engine
        r = getattr(self, 'split_row', None)
        if r is not None and self.rowsplit:
            # a row range of a CSR is a CSR over the same cols / vals arrays: rowptr keeps its absolute offsets
            for a, b in ((0, r), (r, self.shape[0])):
                engine.spmm_csr(self.rowptr[a:b + 1], self.cols, self.vals, X, out[a:b],
                                acc=None if acc is None else acc[a:b], acc_scale=acc_scale, rowsplit=True)
            return out
        return engine.spmm_csr(self.rowptr, self.cols, self.vals, X, out, acc=acc, acc_scale=acc_scale,
                               rowsplit=self.rowsplit)


def sorted_unique_padded(x):
    """The distinct values of an int32 vector as a same-length vector: sorted, every repeat replaced by -1.  Unlike
    torch.unique the length does not depend on the data, so nothing has to be read back by the host."""
    import torch
    s, _ = torch.sort(x)
    s[1:] = torch.where(s[1:] == s[:-1], torch.full_like(s[1:], -1), s[1:])
    return s.int().contiguous()


def batch_rows(u, i, j, num_users, width):
    """The rows of the joint (users; items) table a minibatch of triples touches, as sorted_unique_padded lists them:
    the only rows its losses read and the only rows where their gradients are non-zero.  None when the batch (more than
    8192 triples) or the row width (more than 128) is beyond the row-list kernels."""
    import torch
    if u.shape[0] > 8192 or width > 128:
        return None
    return sorted_unique_padded(torch.cat([u, i + num_users, j + num_users]))


def layer_sum(mats, src, acc, scale, bufs, need=None, nz=None, with_src=True):
    """acc <- scale * (src + A_1 src + A_2 A_1 src + ... + A_n ... A_1 src) for the n operators `mats` (DeviceCSR),
    each layer accumulated in the SpMM epilogue; with_src=False leaves out the src term (acc is zeroed instead).
    bufs: two tables the layers alternate between.  need: the only rows of acc the caller reads -- the last layer,
    whose output feeds no further layer, is then evaluated on those rows alone (from two layers on; the other rows of
    acc lack its term).  nz: the only non-zero rows of src -- the first layer then scatters along their edges.  Row
    lists are sorted, distinct and -1-padded (batch_rows)."""
    from .. import engine
    if with_src:
        engine.axpby(acc, src, src, scale, 0.0)
    else:
        acc.zero_()
    cur, n = src, len(mats)
    for k in range(n):
        nxt = bufs[k % 2]
        if need is not None and k == n - 1 and k > 0:
            mats[k].matmul_rows(cur, need, acc=acc, acc_scale=scale)
            break
        if nz is not None and k == 0:
            mats[k].matmul_sparse_rows(cur, nz, nxt, acc=acc, acc_scale=scale)
        else:
            mats[k].matmul(cur, nxt, acc=acc, acc_scale=scale)
        cur = nxt
    return acc


class GraphRecommender(DeepRecommender):
    def __init__(self, conf, trainingSet, testSet, fold='[1]'):
        super(GraphRecommender, self).__init__(conf, trainingSet, testSet, fold)

    def create_joint_sparse_adjaceny(self):
        n_nodes = self.num_users + self.num_items
        u, i, _ = self.data.training_ids()
        ones = np.ones(u.shape[0], dtype=np.float32)
        upper = sp.csr_matrix((ones, (u, i.astype(np.int64) + self.num_users)), shape=(n_nodes, n_nodes))
        adj = upper + upper.T
        deg = np.asarray(adj.sum(1)).ravel()
        with np.errstate(divide='ignore'):
            d_inv_sqrt = np.power(deg, -0.5)
        d_inv_sqrt[np.isinf(d_inv_sqrt)] = 0.
        scale = sp.diags(d_inv_sqrt)
        return scale.dot(adj).dot(scale)

    def create_joint_sparse_adj_tensor(self):
        """The same matrix as create_joint_sparse_adjaceny(), assembled on the device from the
        id-mapped training pairs (sort + run-length; duplicates summed like scipy's constructor)."""
        import torch
        from ..graph_build import norm_adjacency_csr
        dev = self._device()
        u, i, _ = self.data.training_ids()
        rowptr, cols, vals = norm_adjacency_csr(torch.from_numpy(u), torch.from_numpy(i), self.num_users,
                                                self.num_items, device=dev)
        n = self.num_users + self.num_items
        return DeviceCSR.from_tensors((n, n), rowptr, cols, vals, split_row=self.num_users)

    def create_sparse_rating_matrix(self):
        """(U x I) COO float32, entry = 1/|items rated by the user| (graphRecommender.py:41-51)."""
        u, i, _ = self.data.training_ids()
        per_user = np.array([len(self.data.trainSet_u[self.data.id2user[k]]) for k in range(self.num_users)],
                            dtype=np.float64)
        vals = 1.0 / per_user[u]
        return sp.coo_matrix((vals, (u, i)), shape=(self.num_users, self.num_items), dtype=np.float32)

    def create_sparse_adj_tensor(self):
        return DeviceCSR(self.create_sparse_rating_matrix(), self._device())

    def _export_tables(self, users, items):
        """(U, V) for ranking: propagated user and item rows on the host as float32, cut to emb_size columns."""
        d = self.emb_size
        return users[:, :d].cpu().numpy(), items[:, :d].cpu().numpy()
