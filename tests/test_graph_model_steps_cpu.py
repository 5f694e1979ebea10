"""The engine calls of the LightGCN-family training steps without a GPU: every kernel is replaced by a restatement of its
contract (test_sgl_model_cpu._stub, conftest.row_list_kernel_stand_ins) and wrapped by a recorder that logs each call
with its arguments bound to the engine function's signature -- tensors by the model buffer they live in, everything
else by value.  For LightGCN, SGL (every augmentation type), SimGCL and parallel.ColumnShardedLightGCN at several
depths the log of two steps must equal the call sequence written out below: which kernels run in which order, on
which buffers, with which scales.  Depth 1 is where the row-list gates differ: LightGCN scatters its first backward
layer from the batch's rows at every depth, SGL and SimGCL list rows only from two layers on."""
import contextlib
import inspect
import io
import re

import numpy as np
import pytest

from conftest import row_list_kernel_stand_ins
from qrec_b200.util.config import ModelConf

B = 512                                     # triples per step; row lists are 3B long
SIG = {}                                    # engine signatures, taken before any stand-in replaces them


def _signatures():
    from qrec_b200 import engine as E
    if not SIG:
        SIG.update({n: inspect.signature(f) for n, f in vars(E).items()
                    if inspect.isfunction(f) and f.__module__ == E.__name__ and not n.startswith('_')})


def call(name, *args, **kw):
    """One expected engine call: its arguments bound to the engine signature, defaults filled in."""
    bound = SIG[name].bind(*args, **kw)
    bound.apply_defaults()
    return (name,) + tuple(bound.arguments.items())


class Recorder(object):
    """Wraps every engine function; `log` holds call(...) tuples with the tensors replaced by labels."""

    def __init__(self, monkeypatch, owner):
        import torch
        from qrec_b200 import engine as E
        from qrec_b200.base.graphRecommender import DeviceCSR
        self.torch, self.DeviceCSR, self.owner, self.log, self.named = torch, DeviceCSR, owner, [], {}
        for n in SIG:
            monkeypatch.setattr(E, n, self._wrap(n, getattr(E, n)))

    def _wrap(self, name, fn):
        def rec(*args, **kw):
            bound = SIG[name].bind(*args, **kw)
            bound.apply_defaults()
            self.log.append((name,) + tuple((k, self.label(v)) for k, v in bound.arguments.items()))
            return fn(*args, **kw)
        return rec

    def _buffers(self):
        out = dict(self.named)

        def add(name, v):
            if isinstance(v, self.torch.Tensor) and v._base is None:
                out.setdefault(name, v)
            elif isinstance(v, self.DeviceCSR):
                for part in ('rowptr', 'cols', 'vals'):
                    out.setdefault('%s.%s' % (name, part), getattr(v, part))
            elif isinstance(v, (list, tuple)):
                for k, x in enumerate(v):
                    add('%s%d' % (name, k), x)
            elif isinstance(v, dict):
                for k, x in v.items():
                    add('%s%s' % (name, k), x)
        for name, v in vars(self.owner).items():
            add(name, v)
        return out

    def label(self, v):
        """A tensor inside a model buffer as `name` or `name[row:]`; any other tensor as `tmp[shape]`."""
        if not isinstance(v, self.torch.Tensor):
            return v
        p = v.data_ptr()
        for name, t in self._buffers().items():
            lo = t.data_ptr()
            if lo <= p < lo + t.numel() * t.element_size():
                row = (p - lo) // t.element_size() // (t.stride(0) if t.dim() else 1)
                return name if row == 0 else '%s[%d:]' % (name, row)
        return 'tmp%s' % list(v.shape)


class Csr(object):
    """The engine calls DeviceCSR issues for the operator `name`: split = the row where matmul cuts its launch."""

    def __init__(self, name, split=None):
        self.name, self.split = name, split

    def _arrays(self, row=0):
        rp = '%s.rowptr' % self.name + ('[%d:]' % row if row else '')
        return rp, '%s.cols' % self.name, '%s.vals' % self.name

    def matmul(self, X, Y, acc=None, s=0.0):
        if self.split is None:
            return [call('spmm_csr', *self._arrays(), X, Y, acc=acc, acc_scale=s, rowsplit=True)]
        r = self.split
        return [call('spmm_csr', *self._arrays(), X, Y, acc=acc, acc_scale=s, rowsplit=True),
                call('spmm_csr', *self._arrays(r), X, '%s[%d:]' % (Y, r), acc=None if acc is None else '%s[%d:]' % (acc, r),
                     acc_scale=s, rowsplit=True)]

    def rows(self, X, rows, Y=None, compact=False, acc=None, s=0.0):
        return [call('spmm_csr_rows', *self._arrays(), rows, X, Y, compact=compact, acc=acc, acc_scale=s)]

    def scatter(self, X, rows, Y, acc=None, s=0.0):
        return [call('spmm_csr_scatter_rows', *self._arrays(), rows, X, Y, acc=acc, acc_scale=s)]


ROWS = 'tmp[%d]' % (3 * B)


def layer_mean(mats, src, acc, s, need=None, nz=None, with_src=True, buf='_buf'):
    """acc <- s * (src +) sum_k A_k..A_1 src as the parent's LightGCN / SGL / ColumnShardedLightGCN loops issue it."""
    out = [call('axpby', acc, src, src, s, 0.0)] if with_src else []
    cur, n = src, len(mats)
    for k in range(n):
        nxt = '%s%d' % (buf, k % 2)
        if need is not None and k == n - 1 and k > 0:
            return out + mats[k].rows(cur, need, acc=acc, s=s)
        out += mats[k].scatter(cur, nz, nxt, acc=acc, s=s) if (nz is not None and k == 0) else mats[k].matmul(cur, nxt, acc, s)
        cur = nxt
    return out


def infonce(tab1, tab2, b, d, tau, scale, loss, g1, g2):
    Z, n, S = 'tmp[%d, %d]' % (b, d), 'tmp[%d]' % b, 'tmp[%d, %d]' % (b, b)
    idx = 'tmp[%d]' % b
    return [call('gather_normalize', tab1, idx, Z, n), call('gather_normalize', tab2, idx, Z, n),
            call('sgemm', Z, Z, S, trans_b=True), call('infonce_rows', S, tau, loss),
            call('sgemm', S, Z, Z), call('sgemm', S, Z, Z, trans_a=True),
            call('normalize_bwd_scatter', Z, Z, n, idx, scale, g1), call('normalize_bwd_scatter', Z, Z, n, idx, scale, g2)]


def _model(cls, golden_graph, monkeypatch, tmp_path, section):
    from qrec_b200 import engine as E
    import test_sgl_model_cpu as S
    _signatures()
    S._stub(monkeypatch)
    row_list_kernel_stand_ins(monkeypatch)
    for name in ('bpr_partial_scores', 'bpr_grad_from_scores'):       # only the call sequence matters here
        monkeypatch.setattr(E, name, lambda *a, **k: None)
    monkeypatch.chdir(tmp_path)
    g = golden_graph
    n_tr = 6000
    train = [[u, i, 1.0] for u, i in zip(g['train_users'][:n_tr].tolist(), g['train_items'][:n_tr].tolist())]
    text = re.sub('LightGCN=.*\n', '', str(g['conf']).replace('model.name=LightGCN', 'model.name=' + cls.__name__)
                  .replace('num.factors=64', 'num.factors=10'))
    m = cls(ModelConf.from_string(text + section + '\n'), train, [])
    with contextlib.redirect_stdout(io.StringIO()):
        m.readConfiguration()
        m.initModel()
    return m


def _batches(m, seed):
    import torch
    rng = np.random.default_rng(seed)
    u_all, i_all, _ = m.data.training_ids()
    for _ in range(2):
        pick = rng.choice(len(u_all), B, replace=False)
        u, i = u_all[pick].astype(np.int32), i_all[pick].astype(np.int32)
        j = rng.integers(0, m.num_items, B).astype(np.int32)
        yield tuple(torch.from_numpy(x) for x in (u, i, j))


def _run(rec, step, batches):
    """The recorded log of the steps and, per step, the number of unique users and items of its batch."""
    import torch
    uniq = []
    for u, i, j in batches:
        rec.named.update(u=u, i=i, j=j)
        uniq.append((int(torch.unique(u).numel()), int(torch.unique(i).numel())))
        step(u, i, j)
    return rec.log, uniq


@pytest.mark.parametrize('n', [1, 2, 3])
def test_lightgcn_step_calls(golden_graph, monkeypatch, tmp_path, n):
    from qrec_b200.model.ranking.LightGCN import LightGCN
    m = _model(LightGCN, golden_graph, monkeypatch, tmp_path, 'LightGCN=-n_layer %d' % n)
    nu, s = m.num_users, 1.0 / (n + 1)
    A = [Csr('norm_adj', nu)] * n
    log, _ = _run(Recorder(monkeypatch, m), m.train_step, _batches(m, 5))
    want = []
    for t in (1, 2):
        want += layer_mean(A, 'ego', '_mean', s, need=ROWS)
        want += [call('bpr_grad_scatter', '_mean', '_mean[%d:]' % nu, 'u', 'i', 'j', 10e-8, m.regU, '_grad',
                      '_grad[%d:]' % nu, '_loss')]
        want += layer_mean(A, '_grad', '_total', s, nz=ROWS)
        want += [call('adam_dense_tf1', 'ego', '_adam_m', '_adam_v', '_total', m.lRate, t)]
    assert log == want


@pytest.mark.parametrize('aug', [0, 1, 2])
@pytest.mark.parametrize('n', [1, 2, 3])
def test_sgl_step_calls(golden_graph, monkeypatch, tmp_path, n, aug):
    from qrec_b200.model.ranking.SGL import SGL
    m = _model(SGL, golden_graph, monkeypatch, tmp_path, 'SGL=-n_layer %d -lambda 0.1 -droprate 0.3 -augtype %d -temp 0.2' % (n, aug))
    m.build_views(1)
    nu, d, s = m.num_users, m.emb_pad, 1.0 / (n + 1)
    rows = ROWS if n > 1 else None
    main = [Csr('norm_adj', nu)] * n
    views = [[Csr('views%d%d' % (v, k if aug == 2 else 0), nu) for k in range(n)] for v in (0, 1)]

    def backprop(mats, G):
        out, cur = [], G
        for k in range(n - 1, -1, -1):
            nxt = '_buf%d' % (k % 2)
            out += mats[k].scatter(cur, rows, nxt) if (rows is not None and k == n - 1) else mats[k].matmul(cur, nxt)
            out += [call('axpby', nxt, nxt, G, 1.0, 1.0)]
            cur = nxt
        return out + [call('axpby', '_total', '_total', cur, 1.0, s)]

    log, uniq = _run(Recorder(monkeypatch, m), m.train_step, _batches(m, 6))
    want = []
    for t, (bu, bi) in zip((1, 2), uniq):
        for mats, k in ((main, 0), (views[0], 1), (views[1], 2)):
            want += layer_mean(mats, 'ego', '_mean%d' % k, s, need=rows)
        want += [call('bpr_grad_scatter', '_mean0', '_mean0[%d:]' % nu, 'u', 'i', 'j', 10e-8, m.regU, '_grad0',
                      '_grad0[%d:]' % nu, '_loss')]
        want += infonce('_mean1', '_mean2', bu + bi, d, m.ssl_temp, m.ssl_reg, '_loss[1:]', '_grad1', '_grad2')
        want += backprop(main, '_grad0') + backprop(views[0], '_grad1') + backprop(views[1], '_grad2')
        want += [call('adam_dense_tf1', 'ego', '_adam_m', '_adam_v', '_total', m.lRate, t)]
    assert log == want


@pytest.mark.parametrize('n', [1, 2, 3])
def test_simgcl_step_calls(golden_graph, monkeypatch, tmp_path, n):
    from qrec_b200.model.ranking.SimGCL import SimGCL, TAU
    m = _model(SimGCL, golden_graph, monkeypatch, tmp_path, 'SimGCL=-n_layer %d -lambda 0.5 -eps 0.1' % n)
    nu, d, s = m.num_users, m.emb_pad, 1.0 / n
    rows = ROWS if n > 1 else None
    A = Csr('norm_adj', nu)

    def perturbed(out, view, t):
        res, cur = [], 'ego'
        for k in range(n):
            nxt = '_buf%d' % (k % 2)
            tag = view * 16 + k
            if rows is not None and k == n - 1:
                return res + A.rows(cur, rows, '_rows_buf', compact=True) + [
                    call('simgcl_perturb_listed', '_rows_buf', rows, m.eps, m.noise_seed, tag, t, acc=out, acc_scale=s,
                         d_valid=m.emb_size)]
            res += A.matmul(cur, nxt) + [call('simgcl_perturb', nxt, m.eps, m.noise_seed, tag, t, acc=out, acc_scale=s,
                                              d_valid=m.emb_size)]
            cur = nxt
        return res

    log, uniq = _run(Recorder(monkeypatch, m), m.train_step, _batches(m, 7))
    want = []
    for t, (bu, bi) in zip((1, 2), uniq):
        want += layer_mean([A] * n, 'ego', '_main', s, need=rows, with_src=False)
        want += perturbed('_pert0', 1, t) + perturbed('_pert1', 2, t)
        want += [call('bpr_grad_scatter', '_main', '_main[%d:]' % nu, 'u', 'i', 'j', 10e-8, m.regU, '_grad',
                      '_grad[%d:]' % nu, '_loss')]
        want += infonce('_pert0', '_pert1', bu, d, TAU, m.cl_rate, '_loss[1:]', '_grad', '_grad')
        want += infonce('_pert0[%d:]' % nu, '_pert1[%d:]' % nu, bi, d, TAU, m.cl_rate, '_loss[1:]', '_grad[%d:]' % nu,
                        '_grad[%d:]' % nu)
        want += layer_mean([A] * n, '_grad', '_total', s, nz=rows, with_src=False)
        want += [call('adam_dense_tf1', 'ego', '_adam_m', '_adam_v', '_total', m.lRate, t)]
    assert log == want


@pytest.mark.parametrize('n', [1, 3])
def test_column_sharded_lightgcn_step_calls(golden_graph, monkeypatch, tmp_path, n):
    """parallel.ColumnShardedLightGCN at world size 1 over the FilmTrust joint adjacency (no split row)."""
    import torch
    from qrec_b200 import parallel
    from qrec_b200.base.graphRecommender import DeviceCSR
    from qrec_b200.model.ranking.LightGCN import LightGCN
    shell = _model(LightGCN, golden_graph, monkeypatch, tmp_path, 'LightGCN=-n_layer %d' % n)
    N, nu = shell.num_users + shell.num_items, shell.num_users
    a = shell.norm_adj
    m = parallel.ColumnShardedLightGCN(DeviceCSR.from_tensors((N, N), a.rowptr, a.cols, a.vals), torch.zeros(N, 8), nu, n,
                                       0.001, 0.002)
    s, A = 1.0 / (n + 1), [Csr('adj')] * n
    log, _ = _run(Recorder(monkeypatch, m), m.train_step, _batches(shell, 8))
    want = []
    for t in (1, 2):
        want += layer_mean(A, 'ego', 'mean', s, need=ROWS, buf='buf')
        want += [call('bpr_partial_scores', 'mean', 'mean[%d:]' % nu, 'u', 'i', 'j', 0.002, '_y%d' % B, 'loss'),
                 call('bpr_grad_from_scores', 'mean', 'mean[%d:]' % nu, 'u', 'i', 'j', '_y%d' % B, 10e-8, 0.002, 1.0,
                      'grad', 'grad[%d:]' % nu, 'loss')]
        want += layer_mean(A, 'grad', 'total', s, nz=ROWS, buf='buf')
        want += [call('adam_dense_tf1', 'ego', 'm', 'v', 'total', 0.001, t)]
    assert log == want
