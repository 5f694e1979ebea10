"""NeuMF on the H100 engine -- drop-in for model/ranking/NeuMF.py of the reference.

GMF head + 3-layer MLP (2d -> 5d -> 2d -> d, ReLU) + fused head, trained in the reference's three
phases (GMF `maxEpoch` epochs, MLP `maxEpoch//2`, fused `maxEpoch//5`; NeuMF.py:77-100), each with
its own TF1 Adam optimiser (own slots and step counter) over the variables its loss reaches.
Batches come from next_batch_pointwise (1 positive + 4 sampled negatives per interaction).

Engine mapping (one minibatch of B = 5*batch_size samples):
  gather      qrec_gather_rows_f32 -> UG, IG and the concatenated MLP input [B, 2d]
  MLP fwd     3 x qrec_tc_gemm_tf32 (wgmma TF32, bias+ReLU fused in the epilogue)
  head        qrec_neumf_head_f32: sigmoid, BCE(+1e-9), dz, GMF-side gradients, ReLU-masked dH3
  MLP bwd     dX = dY W^T on the tensor cores (ReLU mask fused); dW = X^T dY and the bias/h-vector
              column sums on the split-K fp32 path (K = B is the long dimension there)
  scatter     qrec_scatter_add_rows_f32 into dense table gradients (duplicates summed, as
              TF sums IndexedSlices) and TF1's non-lazy dense Adam over every reached variable
"""
import math

import numpy as np

from ...base.deepRecommender import DeepRecommender


class NeuMF(DeepRecommender):
    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(NeuMF, self).__init__(conf, trainingSet, testSet, fold)

    # ------------------------------------------------------------------ parameters
    def initModel(self):
        super(NeuMF, self).initModel()
        import torch
        if self.emb_size % 4:
            raise ValueError('NeuMF on the H100 engine needs num.factors to be a multiple of 4 (got %d)' % self.emb_size)
        dev, d = self.device, self.emb_size
        # MLP widths after the 2d-wide input: the reference hard-codes 5d -> 2d -> d (NeuMF.py:39-49); BASELINE.json's
        # config 4 names [256,128,64].  The attribute `mlp_widths` overrides; the last width feeds the fused head
        # together with the d-wide GMF vector (qrec_neumf_head_f32), so it must equal d as in the reference.
        w = getattr(self, 'mlp_widths', None) or (5 * d, 2 * d, d)
        if len(w) != 3 or any(int(x) % 4 for x in w) or int(w[2]) != d:
            raise ValueError('NeuMF: mlp_widths must be three multiples of 4 ending in d=%d, got %r' % (d, w))
        self.mlp_widths = w1, w2, w3 = tuple(int(x) for x in w)
        gen = torch.Generator(device=dev)
        gen.manual_seed(self.engine_seed + 3)

        def xavier(*shape):
            fan_in, fan_out = (shape[0], shape[1]) if len(shape) == 2 else (shape[0], shape[0])
            bound = math.sqrt(6.0 / (fan_in + fan_out))
            return ((torch.rand(*shape, device=dev, generator=gen) * 2 - 1) * bound).contiguous()
        self.params = {
            'PG': xavier(self.num_users, d), 'QG': xavier(self.num_items, d),
            'PM': xavier(self.num_users, d), 'QM': xavier(self.num_items, d),
            'h_mf': xavier(d), 'h_mlp': xavier(w3),
            'W1': xavier(2 * d, w1), 'b1': torch.zeros(w1, device=dev),
            'W2': xavier(w1, w2), 'b2': torch.zeros(w2, device=dev),
            'W3': xavier(w2, w3), 'b3': torch.zeros(w3, device=dev),
        }
        self.grads = {k: torch.zeros_like(v) for k, v in self.params.items()}
        mlp_vars = ['PM', 'QM', 'W1', 'b1', 'W2', 'b2', 'W3', 'b3', 'h_mlp']
        self.opt_vars = {0: ['PG', 'QG', 'h_mf'], 1: mlp_vars, 2: ['PG', 'QG', 'h_mf'] + mlp_vars}
        self.opt_state = {m: {k: (torch.zeros_like(self.params[k]), torch.zeros_like(self.params[k]))
                              for k in self.opt_vars[m]} for m in (0, 1, 2)}
        self.opt_step = {0: 0, 1: 0, 2: 0}
        self._loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self._ws_rows = 0

    def _workspace(self, B):
        import torch
        if B <= self._ws_rows:
            return
        dev, d = self.device, self.emb_size
        w1, w2, w3 = self.mlp_widths
        new = lambda *s: torch.empty(*s, device=dev)          # noqa: E731
        self._UG, self._IG, self._GMF, self._dUG, self._dIG = (new(B, d) for _ in range(5))
        self._X0, self._dX0 = new(B, 2 * d), new(B, 2 * d)
        self._H1, self._dH1 = new(B, w1), new(B, w1)
        self._H2, self._dH2 = new(B, w2), new(B, w2)
        self._H3, self._dH3 = new(B, w3), new(B, w3)
        self._y, self._dz = new(B), new(B)
        self._ones = torch.ones(B, 1, device=dev)
        self._ws_rows = B

    # ------------------------------------------------------------------ forward pieces
    def _forward(self, mode, u, i, B):
        from ... import engine as E
        p, d = self.params, self.emb_size
        if mode != 1:
            E.gather_rows(p['PG'], u, self._UG[:B])
            E.gather_rows(p['QG'], i, self._IG[:B])
        if mode != 0:
            E.gather_rows(p['PM'], u, self._X0[:B, :d])
            E.gather_rows(p['QM'], i, self._X0[:B, d:])
            E.tc_gemm(self._X0[:B], p['W1'], self._H1[:B], epilogue=E.EPI_BIAS_RELU, bias=p['b1'])
            E.tc_gemm(self._H1[:B], p['W2'], self._H2[:B], epilogue=E.EPI_BIAS_RELU, bias=p['b2'])
            E.tc_gemm(self._H2[:B], p['W3'], self._H3[:B], epilogue=E.EPI_BIAS_RELU, bias=p['b3'])

    def train_step(self, mode, u, i, r):
        """One minibatch of phase `mode` (0 GMF, 1 MLP, 2 NeuMF).  u,i: int32 CUDA, r: fp32 CUDA."""
        self._backward(mode, u, i, r)
        return self._update(mode)

    def _backward(self, mode, u, i, r):
        """Forward + loss + the gradient SUMS over the minibatch's samples into self.grads."""
        from ... import engine as E
        p, g, d = self.params, self.grads, self.emb_size
        B = u.shape[0]
        self._workspace(B)
        self._forward(mode, u, i, B)
        self._loss.zero_()
        gm = mode != 1
        ml = mode != 0
        E.neumf_head(mode, 1, self._UG[:B] if gm else None, self._IG[:B] if gm else None,
                     self._H3[:B] if ml else None, p['h_mf'] if gm else None, p['h_mlp'] if ml else None, r,
                     self.regU, self._loss, self._y[:B], self._dz[:B], self._GMF[:B] if gm else None,
                     self._dUG[:B] if gm else None, self._dIG[:B] if gm else None, self._dH3[:B] if ml else None)
        wg = 1.0 if mode == 0 else 0.5
        wm = 1.0 if mode == 1 else 0.5
        for k in self.opt_vars[mode]:
            if g[k].dim() == 2 and g[k].shape[0] in (self.num_users, self.num_items) and k in ('PG', 'QG', 'PM', 'QM'):
                g[k].zero_()
        if gm:
            E.scatter_add_rows(g['PG'], u, self._dUG[:B])
            E.scatter_add_rows(g['QG'], i, self._dIG[:B])
            # d h_mf = wg * GMF^T dz + reg*h_mf (mf_reg) [+ reg*0.25*h_mf: l2_loss(h_NeuMF), mode 2]
            E.gemv_t(self._GMF[:B], self._dz[:B], g['h_mf'], alpha=wg)
        if ml:
            # d h_mlp = wm * relu(H3)^T dz : dH3 already carries wm*dz*h_mlp masked, so use H3 directly
            E.gemv_t(self._H3[:B], self._dz[:B], g['h_mlp'], alpha=wm)
            E.sgemm(self._H2[:B], self._dH3[:B], g['W3'], trans_a=True)
            E.gemv_t(self._dH3[:B], None, g['b3'])
            E.tc_gemm(self._dH3[:B], p['W3'], self._dH2[:B], b_is_nk=True, epilogue=E.EPI_RELU_MASK, mask=self._H2[:B])
            E.sgemm(self._H1[:B], self._dH2[:B], g['W2'], trans_a=True)
            E.gemv_t(self._dH2[:B], None, g['b2'])
            E.tc_gemm(self._dH2[:B], p['W2'], self._dH1[:B], b_is_nk=True, epilogue=E.EPI_RELU_MASK, mask=self._H1[:B])
            E.sgemm(self._X0[:B], self._dH1[:B], g['W1'], trans_a=True)
            E.gemv_t(self._dH1[:B], None, g['b1'])
            E.tc_gemm(self._dH1[:B], p['W1'], self._dX0[:B], b_is_nk=True)
            E.scatter_add_rows(g['PM'], u, self._dX0[:B, :d])
            E.scatter_add_rows(g['QM'], i, self._dX0[:B, d:])

    def _update(self, mode):
        """Parameter-only regularisers + TF1 Adam.  self.grads holds sums over samples: a data-parallel run adds the
        ranks' buffers first (parallel.UserShardedNeuMF._reduce_gradients); the terms added here are applied once."""
        from ... import engine as E
        p, g = self.params, self.grads
        gm, ml = mode != 1, mode != 0
        self._reduce_gradients(mode)
        if gm:
            E.axpby(g['h_mf'], g['h_mf'], p['h_mf'], 1.0, self.regU * (1.25 if mode == 2 else 1.0))
        if ml and mode == 2:
            E.axpby(g['h_mlp'], g['h_mlp'], p['h_mlp'], 1.0, self.regU * 0.25)
        self.opt_step[mode] += 1
        for k in self.opt_vars[mode]:
            m, v = self.opt_state[mode][k]
            E.adam_dense_tf1(p[k], m, v, g[k], self.lRate, self.opt_step[mode])
        return self._loss

    def _reduce_gradients(self, mode):
        """Hook between the per-sample gradient sums and the optimiser; a single process has nothing to add."""

    def loss_value(self, mode):
        """Python float of the last step's loss incl. the h-vector regularisers (NeuMF.py:56-57,72)."""
        import torch
        l = float(self._loss.item())
        p = self.params
        if mode != 1:
            l += self.regU * 0.5 * float((p['h_mf'] ** 2).sum())
        if mode == 2:
            l += self.regU * 0.5 * 0.25 * float((p['h_mf'] ** 2).sum() + (p['h_mlp'] ** 2).sum())
        return l

    def trainModel(self):
        import torch
        phases = ((0, 'pretraining... (GMF)', self.maxEpoch), (1, 'pretraining... (MLP)', self.maxEpoch // 2),
                  (2, 'training... (NeuMF)', self.maxEpoch // 5))
        for mode, banner, epochs in phases:
            print(banner)
            for epoch in range(epochs):
                for num, (u, i, y) in enumerate(self.next_batch_pointwise()):
                    self.train_step(mode, torch.from_numpy(u).to(self.device), torch.from_numpy(i).to(self.device),
                                    torch.from_numpy(y.astype(np.float32)).to(self.device))
                    if num % 20 == 0:
                        print('epoch:', epoch, 'batch:', num, 'loss:', float(self._loss.item()))

    buildModel = trainModel

    # ------------------------------------------------------------------ prediction (NeuMF.py:102-123)
    def _predict(self, mode, uid):
        import torch
        from ... import engine as E
        n = self.num_items
        self._workspace(n)
        u = torch.full((n,), uid, dtype=torch.int32, device=self.device)
        i = torch.arange(n, dtype=torch.int32, device=self.device)
        self._forward(mode, u, i, n)
        p = self.params
        E.neumf_head(mode, 0, self._UG[:n] if mode != 1 else None, self._IG[:n] if mode != 1 else None,
                     self._H3[:n] if mode != 0 else None, p['h_mf'] if mode != 1 else None,
                     p['h_mlp'] if mode != 0 else None, None, 0.0, None, self._y[:n], None, None, None, None, None)
        return self._y[:n].cpu().numpy()

    def predict_mf(self, uid):
        return self._predict(0, uid)

    def predict_mlp(self, uid):
        return self._predict(1, uid)

    def predict_neu(self, uid):
        return self._predict(2, uid)

    def predictForRanking(self, u):
        if self.data.containsUser(u):
            return self.predict_neu(self.data.user[u])
        return [self.data.globalMean] * self.num_items
