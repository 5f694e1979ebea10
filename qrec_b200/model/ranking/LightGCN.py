"""LightGCN on the H100 engine -- drop-in for model/ranking/LightGCN.py of the reference.

The reference re-runs the whole n-layer propagation, its backward pass and a dense Adam update
for EVERY minibatch (LightGCN.py:35-39: one sess.run per batch).  The same computation here:

  forward   E_{k+1} = A E_k (K2 SpMM, layer mean accumulated in the SpMM epilogue)
  loss/grad bpr_loss + batch L2 on the propagated rows, gradient scatter-added (K3)
  backward  dE0 = 1/(n+1) * sum_k A^k G            (A symmetric: the same K2 kernel)
  update    TF1 dense Adam on the ego table        (K4)
"""
from ...base.graphRecommender import GraphRecommender, batch_rows, layer_sum
from ...util.config import OptionConf
from ...util.loss import BPR_EPS


class LightGCN(GraphRecommender):
    score_tables = ('U', 'V')

    def __init__(self, conf, trainingSet=None, testSet=None, fold='[1]'):
        super(LightGCN, self).__init__(conf, trainingSet, testSet, fold)
        args = OptionConf(self.config['LightGCN'])
        self.n_layers = int(args['-n_layer'])

    def initModel(self):
        super(LightGCN, self).initModel()
        import torch
        self.norm_adj = self.create_joint_sparse_adj_tensor()
        n = self.num_users + self.num_items
        # ego table = [U; V] (LightGCN.py:13); user/item_embeddings become views into it
        self.ego = torch.cat([self.user_embeddings, self.item_embeddings], dim=0).contiguous()
        self.user_embeddings = self.ego[:self.num_users]
        self.item_embeddings = self.ego[self.num_users:]
        dev, d = self.device, self.emb_pad
        self._buf = [torch.empty(n, d, device=dev) for _ in range(2)]
        self._mean = torch.empty(n, d, device=dev)
        self._grad = torch.zeros(n, d, device=dev)
        self._total = torch.empty(n, d, device=dev)
        self._adam_m = torch.zeros(n, d, device=dev)
        self._adam_v = torch.zeros(n, d, device=dev)
        self._loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self._step = 0

    def propagate(self, rows=None):
        """mean(E0..En) into self._mean; returns (user rows, item rows) views (LightGCN.py:13-20).
        rows (int32, distinct, -1 padded): the only rows the caller will read -- the last layer, whose output feeds
        no further layer, is then evaluated on those rows alone (the other rows of the mean lack its term)."""
        layer_sum([self.norm_adj] * self.n_layers, self.ego, self._mean, 1.0 / (self.n_layers + 1), self._buf, need=rows)
        return self._mean[:self.num_users], self._mean[self.num_users:]

    def train_step(self, u, i, j):
        """One minibatch (LightGCN.py:28-39).  u,i,j: int32 CUDA tensors.  Returns the device loss."""
        from ... import engine as E
        # listed at every depth: even at one layer the backward pass scatters from the batch's rows
        rows = batch_rows(u, i, j, self.num_users, self.emb_pad)
        Ue, Ve = self.propagate(rows)
        self._grad.zero_()
        self._loss.zero_()
        E.bpr_grad_scatter(Ue, Ve, u, i, j, BPR_EPS, self.regU, self._grad[:self.num_users],
                           self._grad[self.num_users:], self._loss)
        # dE0 = 1/(n+1) sum_k A^k G (A symmetric); G is non-zero only in the batch's rows
        layer_sum([self.norm_adj] * self.n_layers, self._grad, self._total, 1.0 / (self.n_layers + 1), self._buf, nz=rows)
        self._step += 1
        E.adam_dense_tf1(self.ego, self._adam_m, self._adam_v, self._total, self.lRate, self._step)
        return self._loss

    def trainModel(self):
        import torch
        for epoch in range(self.maxEpoch):
            for n, (u, i, j) in enumerate(self.next_batch_pairwise()):
                loss = self.train_step(torch.from_numpy(u).to(self.device), torch.from_numpy(i).to(self.device),
                                       torch.from_numpy(j).to(self.device))
                if n % 20 == 0:      # the reference prints every batch; rate-limited here
                    print(self.foldInfo, 'training:', epoch + 1, 'batch', n, 'loss:', float(loss.item()))
        self.U, self.V = self._export_tables(*self.propagate())

    buildModel = trainModel

    def device_tables(self):
        return self._tables_on_device()
