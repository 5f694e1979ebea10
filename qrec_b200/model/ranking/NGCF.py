"""NGCF on the H100 engine -- drop-in for model/ranking/NGCF.py of the reference.

Two propagation layers (hard-coded in the reference, NGCF.py:19); per layer
    side = A ego                                   K2 SpMM
    Z    = (side + ego) W1 + (ego * side) W2       qrec_sgemm_f32 (x2) + qrec_mul_f32
    ego' = dropout_0.9(leaky_relu_0.2(Z))          qrec_ngcf_act_fwd_f32 (training only)
    out  = l2_normalize(ego')
and the final table is concat[E0, out_1, out_2] ([N, 3d], NGCF.py:42).  The reference re-runs all
of this and its TF-generated backward pass for every minibatch; the backward pass here is derived
by hand (checked against torch autograd in tests/test_gpu_models.py) and reuses the same kernels.
"""
import math

from ...base.graphRecommender import GraphRecommender
from ...util.loss import BPR_EPS

KEEP_PROB = 0.9           # NGCF.py:37


class NGCF(GraphRecommender):
    score_tables = ('U', 'V')

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(NGCF, self).__init__(conf, trainingSet, testSet, fold)

    def initModel(self):
        super(NGCF, self).initModel()
        import torch
        if self.emb_size % 4:
            raise ValueError('NGCF on the H100 engine needs num.factors to be a multiple of 4 (got %d)' % self.emb_size)
        dev, d = self.device, self.emb_size
        self.n_layers = 2
        n = self.num_users + self.num_items
        gen = torch.Generator(device=dev)
        gen.manual_seed(self.engine_seed + 2)
        bound = math.sqrt(6.0 / (d + d))                      # xavier_initializer on [d, d]
        self.weights = {}
        for k in range(self.n_layers):
            for w in (1, 2):
                self.weights['W_%d_%d' % (k, w)] = ((torch.rand(d, d, device=dev, generator=gen) * 2 - 1) * bound).contiguous()
        self.ego = torch.cat([self.user_embeddings, self.item_embeddings], dim=0).contiguous()
        self.user_embeddings, self.item_embeddings = self.ego[:self.num_users], self.ego[self.num_users:]
        self.norm_adj = self.create_joint_sparse_adj_tensor()
        new = lambda *shape: torch.empty(*shape, device=dev)          # noqa: E731
        self._side = [new(n, d) for _ in range(self.n_layers)]
        self._Z = [new(n, d) for _ in range(self.n_layers)]
        self._H = [new(n, d) for _ in range(self.n_layers)]
        self._norms = [new(n) for _ in range(self.n_layers)]
        self._all = new(n, (self.n_layers + 1) * d)
        self._gall = torch.zeros(n, (self.n_layers + 1) * d, device=dev)
        self._t1, self._t2, self._dz = new(n, d), new(n, d), new(n, d)
        self._dside, self._dego, self._tmp = new(n, d), new(n, d), new(n, d)
        self._gw = {k: torch.zeros_like(v) for k, v in self.weights.items()}
        self._adam = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in list(self.weights.items()) + [('ego', self.ego)]}
        self._loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self._step = 0
        self.noise_seed = self.engine_seed + 0x6e67

    def forward(self, training):
        """Fills self._all ([N, 3d]) and the per-layer caches; returns (user rows, item rows)."""
        from ... import engine as E
        d = self.emb_size
        self._all[:, :d].copy_(self.ego)
        ego = self.ego
        for k in range(self.n_layers):
            side = self._side[k]
            self.norm_adj.matmul(ego, side)
            E.axpby(self._t1, side, ego, 1.0, 1.0)
            E.mul(self._t2, ego, side)
            E.sgemm(self._t1, self.weights['W_%d_1' % k], self._Z[k])
            E.sgemm(self._t2, self.weights['W_%d_2' % k], self._Z[k], beta=1.0)
            E.ngcf_act_fwd(self._Z[k], KEEP_PROB, training, self.noise_seed, k, self._step, self._H[k],
                           self._all[:, (k + 1) * d:(k + 2) * d], self._norms[k])
            ego = self._H[k]
        return self._all[:self.num_users], self._all[self.num_users:]

    def train_step(self, u, i, j):
        from ... import engine as E
        d, nu = self.emb_size, self.num_users
        self._step += 1
        Ue, Ve = self.forward(1)
        self._gall.zero_()
        self._loss.zero_()
        E.bpr_grad_scatter(Ue, Ve, u, i, j, BPR_EPS, self.regU, self._gall[:nu], self._gall[nu:], self._loss)
        dH_extra = None
        for k in reversed(range(self.n_layers)):
            ego_in = self.ego if k == 0 else self._H[k - 1]
            side = self._side[k]
            E.ngcf_act_bwd(self._gall[:, (k + 1) * d:(k + 2) * d], dH_extra, self._H[k], self._Z[k], self._norms[k],
                           KEEP_PROB, 1, self.noise_seed, k, self._step, self._dz)
            E.axpby(self._t1, side, ego_in, 1.0, 1.0)
            E.mul(self._t2, ego_in, side)
            E.sgemm(self._t1, self._dz, self._gw['W_%d_1' % k], trans_a=True)          # dW1 = (side+ego)^T dZ
            E.sgemm(self._t2, self._dz, self._gw['W_%d_2' % k], trans_a=True)          # dW2 = (ego*side)^T dZ
            E.sgemm(self._dz, self.weights['W_%d_1' % k], self._t1, trans_b=True)      # dT1 = dZ W1^T
            E.sgemm(self._dz, self.weights['W_%d_2' % k], self._t2, trans_b=True)      # dT2 = dZ W2^T
            E.mul(self._tmp, self._t2, ego_in)
            E.axpby(self._dside, self._t1, self._tmp, 1.0, 1.0)                        # d side = dT1 + dT2*ego
            E.mul(self._tmp, self._t2, side)
            E.axpby(self._dego, self._t1, self._tmp, 1.0, 1.0)                         # d ego  = dT1 + dT2*side ...
            self.norm_adj.matmul(self._dside, self._tmp, acc=self._dego, acc_scale=1.0)  # ... + A d side
            dH_extra = self._dego
        # gradient of the E0 block of the concatenation
        E.axpby(self._dego, self._dego, self._gall[:, :d].contiguous(), 1.0, 1.0)
        m, v = self._adam['ego']
        E.adam_dense_tf1(self.ego, m, v, self._dego, self.lRate, self._step)
        for name, w in self.weights.items():
            m, v = self._adam[name]
            E.adam_dense_tf1(w, m, v, self._gw[name], self.lRate, self._step)
        return self._loss

    def trainModel(self):
        import torch
        for epoch in range(self.maxEpoch):
            for n, (u, i, j) in enumerate(self.next_batch_pairwise()):
                loss = self.train_step(*(torch.from_numpy(x).to(self.device) for x in (u, i, j)))
                if n % 20 == 0:
                    print('training:', epoch + 1, 'batch', n, 'loss:', float(loss.item()))
        Ue, Ve = self.forward(0)                    # inference: no dropout (NGCF.py:70)
        self.U, self.V = Ue.cpu().numpy(), Ve.cpu().numpy()

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
