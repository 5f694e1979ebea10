"""SGL (self-supervised graph learning) on the H100 engine -- drop-in for model/ranking/SGL.py of the reference.

Per epoch the reference rebuilds two augmented views of the interaction graph on the host with scipy
(`_create_adj_mat`, SGL.py:113-155; aug_type 0 node dropout, 1 edge dropout, 2 "random walk" = a fresh edge
dropout per layer) and feeds them as SparseTensors; per minibatch it runs three LightGCN encoders (full graph, view
1, view 2; mean of E_0..E_n), BPR + batch L2 on the full-graph one, the merged user+item InfoNCE of
`calc_ssl_loss_v3` between the two views (SGL.py:206-230) and a dense Adam step (SGL.py:232-283).  Here:

  views      graph_build.JointAdjacency.edge_dropout: Philox keep flags per interaction line -> multiplicities ->
             kept counts, degrees, scan, ordered compaction with the sub-graph's own D^-1/2 (csrc/adj_kernels.cu);
             node dropout masks the lines of the dropped users / items and goes through the same rebuild.
             The reference draws `random.sample` (exact count) from Python's generator; the engine's views are
             Bernoulli(1 - rate) per line from a Philox stream keyed (seed, view, epoch[, layer]).
  encoders   K2 SpMM per layer with the layer mean fused into the epilogue
  losses     K3 (bpr_loss + batch L2), gather_normalize / sgemm / infonce_rows / normalize_bwd_scatter (K6)
  backward   each encoder is linear in E_0: d/dE_0 = 1/(n+1) (G + A_1 (G + A_2 (... + A_n G))) per view (Horner)
  update     TF1 dense Adam (K4) on the ego table
"""
from ...base.graphRecommender import GraphRecommender, DeviceCSR, batch_rows, layer_sum
from ...util.config import OptionConf
from ...util.loss import BPR_EPS, infonce_step


class SGL(GraphRecommender):
    score_tables = ('U', 'V')

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(SGL, self).__init__(conf, trainingSet, testSet, fold)

    def readConfiguration(self):
        super(SGL, self).readConfiguration()
        args = OptionConf(self.config['SGL'])
        self.ssl_reg = float(args['-lambda'])
        self.drop_rate = float(args['-droprate'])
        self.aug_type = int(args['-augtype'])
        self.ssl_temp = float(args['-temp'])
        self.n_layers = int(args['-n_layer'])

    def initModel(self):
        super(SGL, self).initModel()
        import torch
        from ...graph_build import JointAdjacency
        dev, d = self.device, self.emb_pad
        n = self.num_users + self.num_items
        u, i, _ = self.data.training_ids()
        self.joint = JointAdjacency(torch.from_numpy(u), torch.from_numpy(i), self.num_users, self.num_items, device=dev)
        self._lines_u = torch.from_numpy(u).to(dev).long()
        self._lines_i = torch.from_numpy(i).to(dev).long()
        self.norm_adj = DeviceCSR.from_tensors((n, n), *self.joint.full(), split_row=self.num_users)
        self.ego = torch.cat([self.user_embeddings, self.item_embeddings], dim=0).contiguous()
        self.user_embeddings = self.ego[:self.num_users]
        self.item_embeddings = self.ego[self.num_users:]
        z = lambda: torch.zeros(n, d, device=dev)                 # noqa: E731
        self._buf = [z(), z()]
        self._mean = [z(), z(), z()]                               # main, view 1, view 2
        self._grad = [z(), z(), z()]
        self._total = z()
        self._adam_m, self._adam_v = z(), z()
        self._loss = torch.zeros(2, dtype=torch.float64, device=dev)   # [rec, ssl (unscaled)]
        self._step = 0
        self.aug_seed = self.engine_seed + 0x5617
        self.views = None

    # ------------------------------------------------------------------ augmented views (SGL.py:113-155, 233-250)
    def build_views(self, epoch):
        """[[A_1..A_n] for view 1, [...] for view 2] as DeviceCSR; aug 0/1 share one sub-graph across layers."""
        import torch
        n = self.num_users + self.num_items
        views = []
        for v in (1, 2):
            mats = []
            for k in range(self.n_layers if self.aug_type == 2 else 1):
                tag = v * 64 + k
                if self.aug_type == 0:                                   # node dropout: lines of dropped users / items go
                    g = torch.Generator(device=self.device)
                    g.manual_seed((self.aug_seed * 1000003 + epoch * 131 + tag) & 0x7fffffff)
                    keep_u = torch.rand(self.num_users, device=self.device, generator=g) >= self.drop_rate
                    keep_i = torch.rand(self.num_items, device=self.device, generator=g) >= self.drop_rate
                    keep = (keep_u[self._lines_u] & keep_i[self._lines_i]).to(torch.uint8).contiguous()
                    csr = self.joint.edge_dropout(self.drop_rate, self.aug_seed, tag, epoch, keep=keep)
                else:
                    csr = self.joint.edge_dropout(self.drop_rate, self.aug_seed, tag, epoch)
                mats.append(DeviceCSR.from_tensors((n, n), *csr, split_row=self.num_users))
            views.append(mats * self.n_layers if len(mats) == 1 else mats)
        self.views = views
        return views

    # ------------------------------------------------------------------ encoders
    def encode(self, mats, out, rows=None):
        """out <- mean(E_0, A_1 E_0, A_2 A_1 E_0, ...) (SGL.py:56-76).
        rows (int32, distinct, -1 padded): the only rows of `out` the caller reads -- the last layer is then
        evaluated on those rows alone (the other rows of `out` lack its term)."""
        return layer_sum(mats, self.ego, out, 1.0 / (self.n_layers + 1), self._buf, need=rows)

    def _backprop(self, mats, G, rows=None):
        """self._total += 1/(n+1) (G + A_1 (G + A_2 (... + A_n G))): the encoder's transpose (A symmetric).
        rows: the only non-zero rows of G -- the innermost product scatters along those rows' edges."""
        from ... import engine as E
        s = 1.0 / (self.n_layers + 1)
        cur = G
        for k in range(self.n_layers - 1, -1, -1):
            nxt = self._buf[k % 2]
            if rows is not None and k == self.n_layers - 1:
                mats[k].matmul_sparse_rows(cur, rows, nxt)
            else:
                mats[k].matmul(cur, nxt)
            E.axpby(nxt, nxt, G, 1.0, 1.0)
            cur = nxt
        E.axpby(self._total, self._total, cur, 1.0, s)

    def train_step(self, u, i, j):
        """One minibatch (SGL.py:232-283).  self._loss holds [rec, ssl_unscaled] afterwards."""
        import torch
        from ... import engine as E
        nu, d = self.num_users, self.emb_pad
        main_mats = [self.norm_adj] * self.n_layers
        self._step += 1
        # the rows the batch touches: all the losses read of the encoders' outputs, and the only rows where their
        # gradients are non-zero; listed from two layers on
        rows = batch_rows(u, i, j, nu, d) if self.n_layers > 1 else None
        m0 = self.encode(main_mats, self._mean[0], rows)
        m1 = self.encode(self.views[0], self._mean[1], rows)
        m2 = self.encode(self.views[1], self._mean[2], rows)
        for g in self._grad:
            g.zero_()
        self._loss.zero_()
        E.bpr_grad_scatter(m0[:nu], m0[nu:], u, i, j, BPR_EPS, self.regU, self._grad[0][:nu], self._grad[0][nu:], self._loss[0:1])
        # calc_ssl_loss_v3: users and items of the batch in ONE InfoNCE (SGL.py:206-230)
        idx = torch.cat([torch.unique(u), torch.unique(i) + nu]).int().contiguous()
        infonce_step(m1, m2, idx, self.ssl_temp, self.ssl_reg, self._loss[1:2], self._grad[1], self._grad[2])
        self._total.zero_()
        self._backprop(main_mats, self._grad[0], rows)
        self._backprop(self.views[0], self._grad[1], rows)
        self._backprop(self.views[1], self._grad[2], rows)
        E.adam_dense_tf1(self.ego, self._adam_m, self._adam_v, self._total, self.lRate, self._step)
        return self._loss

    def losses(self):
        l = self._loss.cpu().numpy()
        return float(l[0]), self.ssl_reg * float(l[1])

    def saveModel(self):
        m0 = self.encode([self.norm_adj] * self.n_layers, self._mean[0])
        self.bestU, self.bestV = self._export_tables(m0[:self.num_users], m0[self.num_users:])

    def trainModel(self):
        import torch
        for epoch in range(self.maxEpoch):
            self.build_views(epoch)
            for n, (u, i, j) in enumerate(self.next_batch_pairwise()):
                self.train_step(*(torch.from_numpy(x).to(self.device) for x in (u, i, j)))
                if n % 20 == 0:
                    rec, ssl = self.losses()
                    print('training:', epoch + 1, 'batch', n, 'rec_loss:', rec, 'ssl_loss', ssl)
            m0 = self.encode([self.norm_adj] * self.n_layers, self._mean[0])
            self.U, self.V = self._export_tables(m0[:self.num_users], m0[self.num_users:])
            self.ranking_performance(epoch)
        self.U, self.V = self.bestU, self.bestV

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
