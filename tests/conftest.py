import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a box without a GPU skips the gpu-marked tests instead of failing them."""
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:                                    # noqa: BLE001
        has_cuda = False
    if has_cuda:
        # `pytest -x` stops at the first failure: run the suites with the longest hardware record first and the ones
        # added most recently last, so that a regression in new code cannot hide the evidence for the old
        late = ['lifecycle[SGL']
        rank = lambda it: next((k + 1 for k, name in enumerate(late) if name in it.nodeid), 0)   # noqa: E731
        items.sort(key=rank)                         # stable: everything else keeps its order
        return
    skip = pytest.mark.skip(reason='needs a CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_bpr():
    return np.load(os.path.join(GOLDEN, 'bpr_filmtrust_seed0.npz'))


@pytest.fixture(scope='session')
def golden_graph():
    return np.load(os.path.join(GOLDEN, 'sampler_graph_filmtrust_seed1234.npz'))


def ids_from_names(names, vocab):
    lut = {n: k for k, n in enumerate(vocab.tolist())}
    return np.array([lut[n] for n in names.tolist()], dtype=np.int32)


@pytest.fixture(scope='session')
def bpr_ids(golden_bpr):
    """(u_ids, i_ids, num_users, num_items) of the FilmTrust training list in reference order."""
    g = golden_bpr
    u = ids_from_names(g['train_users'], g['user_names'])
    i = ids_from_names(g['train_items'], g['item_names'])
    return u, i, len(g['user_names']), len(g['item_names'])


@pytest.fixture(scope='session')
def graph_ids(golden_graph):
    g = golden_graph
    u = ids_from_names(g['train_users'], g['user_names'])
    i = ids_from_names(g['train_items'], g['item_names'])
    return u, i, len(g['user_names']), len(g['item_names'])


def rows_and_sets(u, i, num_users):
    """dict-of-dict view of the training list: per-user item lists (insertion order, dedup) + sets."""
    rows = [dict() for _ in range(num_users)]
    for uu, ii in zip(u.tolist(), i.tolist()):
        rows[uu][ii] = 1
    return [list(r.keys()) for r in rows], [set(r.keys()) for r in rows]


def adjacency_kernel_stand_ins(monkeypatch):
    """numpy restatements of the two value kernels of csrc/adj_kernels.cu (the GPU suite runs the real ones)."""
    import torch
    from qrec_b200 import engine as E

    def line_weights(line_pair, keep, pair_w):
        k = np.ones(len(line_pair), bool) if keep is None else keep.numpy().astype(bool)
        pair_w.copy_(torch.from_numpy(np.bincount(line_pair.numpy()[k], minlength=len(pair_w)).astype(np.float32)))
        return pair_w

    def normalize(rowptr, cols, pair, pair_w, deg, vals):
        rp, co = rowptr.numpy(), cols.numpy()
        w = pair_w.numpy()[pair.numpy()]
        row = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
        d = np.zeros(len(rp) - 1, np.float32)
        np.add.at(d, row, w)
        with np.errstate(divide='ignore'):
            dinv = np.where(d > 0, (1.0 / np.sqrt(d.astype(np.float64))), 0.0).astype(np.float32)
        deg.copy_(torch.from_numpy(d))
        vals.copy_(torch.from_numpy((dinv[row] * w) * dinv[co]))
        return vals
    monkeypatch.setattr(E, 'adj_line_weights', line_weights)
    monkeypatch.setattr(E, 'adj_normalize', normalize)


def row_list_kernel_stand_ins(monkeypatch):
    """numpy / torch restatements of the contracts of the row-list kernels (include/qrec.h: qrec_spmm_csr_rows_f32,
    qrec_spmm_csr_scatter_rows_f32, qrec_simgcl_perturb_{rows,listed}_f32, qrec_scatter_add_rows_f32) for the CPU
    tests of the classes that compose them.  Each stand-in asserts the caller's side of the contract (distinct
    listed rows; the source is zero outside the listed rows)."""
    import numpy as np
    import scipy.sparse as sp
    import torch
    from oracle import tf_models
    from qrec_b200 import engine as E
    calls = []

    def dense(rowptr, cols, vals, n_cols):
        # a row range of a CSR is passed as a slice of rowptr over the whole cols / vals arrays (absolute offsets)
        rp = rowptr.numpy()
        a, b = int(rp[0]), int(rp[-1])
        return sp.csr_matrix((vals.numpy()[a:b], cols.numpy()[a:b], rp - a), shape=(rowptr.numel() - 1, n_cols))

    def listed(rows):
        got = rows[rows >= 0].long()
        assert got.numel() == torch.unique(got).numel(), 'listed rows must be distinct'
        return got

    def spmm_rows(rowptr, cols, vals, rows, X, Y=None, compact=False, acc=None, acc_scale=0.0):
        calls.append('rows')
        got = listed(rows)
        part = torch.from_numpy(np.asarray(dense(rowptr, cols, vals, X.shape[0])[got.numpy()] @ X.numpy())).float()
        if Y is not None:
            if compact:
                Y.zero_()
                Y[(rows >= 0).nonzero().ravel()] = part
            else:
                Y[got] = part
        if acc is not None:
            acc[got] += acc_scale * part
        return Y

    def scatter_rows(rowptr, cols, vals, src_rows, X, Y, acc=None, acc_scale=0.0):
        calls.append('scatter_rows')
        keep = torch.zeros(X.shape[0], dtype=torch.bool)
        keep[listed(src_rows)] = True
        assert float(X[~keep].abs().sum()) == 0.0, 'the source must be zero outside the listed rows'
        Y.copy_(torch.from_numpy(np.asarray(dense(rowptr, cols, vals, Y.shape[0]).T @ X.numpy())).float())
        if acc is not None:
            acc.add_(Y, alpha=acc_scale)
        return Y

    def _noise(n_rows, d, seed, tag, step, d_valid):
        nz = torch.from_numpy(tf_models.philox_uniform(n_rows, d, seed, tag, step)).float()
        if 0 < d_valid < d:
            nz[:, d_valid:] = 0.0
        return nz / nz.norm(dim=1, keepdim=True).clamp(min=1e-6)

    def perturb(Emb, eps, seed, tag, step, acc=None, acc_scale=0.0, d_valid=0, row_offset=0):
        nz = _noise(row_offset + Emb.shape[0], Emb.shape[1], seed, tag, step, d_valid)[row_offset:]
        Emb.add_(torch.sign(Emb) * nz * eps)
        if acc is not None:
            acc.add_(Emb, alpha=acc_scale)
        return Emb

    def perturb_listed(Ec, rows, eps, seed, tag, step, acc=None, acc_scale=0.0, d_valid=0, row_offset=0):
        calls.append('perturb_listed')
        got, slots = listed(rows), (rows >= 0).nonzero().ravel()
        nz = _noise(row_offset + int(got.max()) + 1 if got.numel() else 1, Ec.shape[1], seed, tag, step, d_valid)
        Ec[slots] = Ec[slots] + torch.sign(Ec[slots]) * nz[row_offset + got] * eps
        if acc is not None:
            acc[got] += acc_scale * Ec[slots]
        return Ec

    def scatter_add_rows(G, idx, src, scale=1.0):
        ok = idx >= 0
        G.index_add_(0, idx[ok].long(), scale * src[ok])
        return G

    def gather_rows(T, idx, out):
        ok = idx >= 0
        out.zero_()
        out[ok] = T[idx[ok].long()]
        return out

    for name, fn in (('spmm_csr_rows', spmm_rows), ('spmm_csr_scatter_rows', scatter_rows), ('simgcl_perturb', perturb),
                     ('simgcl_perturb_listed', perturb_listed), ('scatter_add_rows', scatter_add_rows), ('gather_rows', gather_rows)):
        monkeypatch.setattr(E, name, fn)
    return calls
