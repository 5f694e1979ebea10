"""SimGCL on the H100 engine -- drop-in for model/ranking/SimGCL.py of the reference.

Per minibatch the reference runs three LightGCN encoders over the whole graph (one clean, two with
fresh uniform-noise perturbation after every layer), BPR + batch L2 on the clean one, InfoNCE
(tau = 0.2) between the two perturbed views on the batch's unique users and items, and a dense
Adam step (SimGCL.py:22-38, 60-111).  Here:

  encoders   K2 SpMM per layer; the perturbed ones add sign(E) * l2_normalize(noise) * eps with
             Philox noise generated in registers (qrec_simgcl_perturb_f32), layer mean fused in
  losses     K3 (bpr_loss + batch L2) and the K6 InfoNCE kernels, all gradients land in ONE dense
             buffer: d/dE0 of every encoder is the same linear map 1/n * sum_k A^k (the noise is
             additive and tf.sign has zero gradient), so the three backward passes collapse to one
  update     TF1 dense Adam (K4) on the ego table
"""
import math

from ...base.graphRecommender import GraphRecommender, batch_rows, layer_sum
from ...util.config import OptionConf
from ...util.loss import BPR_EPS, infonce_step

TAU = 0.2                      # the literal in SimGCL.py:72-75


class SimGCL(GraphRecommender):
    score_tables = ('U', 'V')

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(SimGCL, self).__init__(conf, trainingSet, testSet, fold)

    def readConfiguration(self):
        super(SimGCL, self).readConfiguration()
        args = OptionConf(self.config['SimGCL'])
        self.cl_rate = float(args['-lambda'])
        self.eps = float(args['-eps'])
        self.n_layers = int(args['-n_layer'])

    @staticmethod
    def xavier_uniform(rows, cols, device, generator=None):
        """tf.contrib.layers.xavier_initializer() (uniform): U(+-sqrt(6/(fan_in+fan_out))) with
        fan_in = rows, fan_out = cols for a [rows, cols] table."""
        import torch
        bound = math.sqrt(6.0 / (rows + cols))
        return (torch.rand(rows, cols, device=device, generator=generator) * 2 - 1) * bound

    def initModel(self):
        super(SimGCL, self).initModel()
        import torch
        dev, d = self.device, self.emb_pad
        gen = torch.Generator(device=dev)
        gen.manual_seed(self.engine_seed + 1)
        n = self.num_users + self.num_items
        self.ego = torch.cat([self.pad_columns(self.xavier_uniform(self.num_users, self.emb_size, dev, gen)),
                              self.pad_columns(self.xavier_uniform(self.num_items, self.emb_size, dev, gen))], dim=0).contiguous()
        self.user_embeddings = self.ego[:self.num_users]       # SimGCL.py:43-44 replaces the base tables
        self.item_embeddings = self.ego[self.num_users:]
        self.norm_adj = self.create_joint_sparse_adj_tensor()
        self._buf = [torch.empty(n, d, device=dev) for _ in range(2)]
        self._main = torch.empty(n, d, device=dev)
        self._pert = [torch.empty(n, d, device=dev) for _ in range(2)]
        self._grad = torch.zeros(n, d, device=dev)
        self._total = torch.zeros(n, d, device=dev)
        self._adam_m = torch.zeros(n, d, device=dev)
        self._adam_v = torch.zeros(n, d, device=dev)
        self._loss = torch.zeros(2, dtype=torch.float64, device=dev)      # [rec, cl]
        self._step = 0
        self.noise_seed = self.engine_seed + 0x5151

    # ------------------------------------------------------------------ encoders
    def encode(self, out, perturbed=0, rows=None):
        """mean(E_1..E_n) into `out` (E0 excluded: SimGCL.py:23-28).  perturbed = 0 | 1 | 2.
        rows (int32, distinct, -1 padded): the only rows of `out` the caller reads -- the last layer (product and
        noise) is then evaluated on those rows alone; the other rows of `out` lack its term."""
        from ... import engine as E
        s = 1.0 / self.n_layers
        if not perturbed:
            layer_sum([self.norm_adj] * self.n_layers, self.ego, out, s, self._buf, need=rows, with_src=False)
            return out[:self.num_users], out[self.num_users:]
        out.zero_()
        cur = self.ego
        for k in range(self.n_layers):
            nxt = self._buf[k % 2]
            if rows is not None and k == self.n_layers - 1 and k > 0:
                part = self._rows_block(rows.shape[0])
                self.norm_adj.matmul_rows(cur, rows, out=part, compact=True)
                E.simgcl_perturb_listed(part, rows, self.eps, self.noise_seed, perturbed * 16 + k, self._step, acc=out,
                                        acc_scale=s, d_valid=self.emb_size)
                break
            self.norm_adj.matmul(cur, nxt)
            E.simgcl_perturb(nxt, self.eps, self.noise_seed, perturbed * 16 + k, self._step, acc=out, acc_scale=s,
                             d_valid=self.emb_size)
            cur = nxt
        return out[:self.num_users], out[self.num_users:]

    def _rows_block(self, n):
        import torch
        if getattr(self, '_rows_buf', None) is None or self._rows_buf.shape[0] < n:
            self._rows_buf = torch.empty(n, self.emb_pad, device=self.device)
        return self._rows_buf[:n]

    def train_step(self, u, i, j):
        """One minibatch (SimGCL.py:92-108).  Returns (total, rec, cl) losses as floats lazily:
        the device tensor self._loss holds [rec, cl_unscaled]."""
        import torch
        from ... import engine as E
        nu = self.num_users
        self._step += 1
        # the rows the batch touches: every loss term reads the encoders' outputs there and nowhere else, and the
        # summed loss gradient is zero everywhere else; listed from two layers on
        rows = batch_rows(u, i, j, nu, self.emb_pad) if self.n_layers > 1 else None
        mU, mV = self.encode(self._main, 0, rows)
        p1U, p1V = self.encode(self._pert[0], 1, rows)
        p2U, p2V = self.encode(self._pert[1], 2, rows)
        self._grad.zero_()
        self._loss.zero_()
        E.bpr_grad_scatter(mU, mV, u, i, j, BPR_EPS, self.regU, self._grad[:nu], self._grad[nu:], self._loss[0:1])
        uu = torch.unique(u).int()                                # tf.unique (order is irrelevant to the sums)
        ii = torch.unique(i).int()
        infonce_step(p1U, p2U, uu, TAU, self.cl_rate, self._loss[1:2], self._grad[:nu], self._grad[:nu])
        infonce_step(p1V, p2V, ii, TAU, self.cl_rate, self._loss[1:2], self._grad[nu:], self._grad[nu:])
        # backward through the encoders: total = 1/n * sum_{k=1..n} A^k G
        layer_sum([self.norm_adj] * self.n_layers, self._grad, self._total, 1.0 / self.n_layers, self._buf, nz=rows,
                  with_src=False)
        E.adam_dense_tf1(self.ego, self._adam_m, self._adam_v, self._total, self.lRate, self._step)
        return self._loss

    def losses(self):
        l = self._loss.cpu().numpy()
        rec, cl = float(l[0]), self.cl_rate * float(l[1])
        return rec + cl, rec, cl

    def saveModel(self):
        self.bestU, self.bestV = self._export_tables(*self.encode(self._main, 0))

    def trainModel(self):
        import torch
        for epoch in range(self.maxEpoch):
            for n, (u, i, j) in enumerate(self.next_batch_pairwise()):
                self.train_step(*(torch.from_numpy(x).to(self.device) for x in (u, i, j)))
                if n % 20 == 0:
                    total, rec, cl = self.losses()
                    print('training:', epoch + 1, 'batch', n, 'total_loss:', total, 'rec_loss:', rec, 'cl_loss', cl)
            self.U, self.V = self._export_tables(*self.encode(self._main, 0))
            self.ranking_performance(epoch)
        self.U, self.V = self.bestU, self.bestV

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
