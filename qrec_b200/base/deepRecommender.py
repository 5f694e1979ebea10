"""`DeepRecommender`: fp32 device tables + the two minibatch samplers of the TF-style models
(reference: base/deepRecommender.py:9-77), without TensorFlow.

* `user_embeddings` / `item_embeddings` are torch CUDA tensors initialised like
  tf.truncated_normal(stddev=0.005) (mean 0, redrawn outside +-2 sigma).
* `next_batch_pairwise` / `next_batch_pointwise` yield int32 numpy arrays instead of Python lists;
  the values are the reference's, bit for bit: the shuffle and every `choice`/`randint` draw go
  through the C MT19937 clone, which continues from (and hands back) the interpreter's global
  `random` state.
"""
import random

from .iterativeRecommender import IterativeRecommender


class DeepRecommender(IterativeRecommender):
    def __init__(self, conf, trainingSet, testSet, fold='[1]'):
        super(DeepRecommender, self).__init__(conf, trainingSet, testSet, fold)

    def readConfiguration(self):
        super(DeepRecommender, self).readConfiguration()
        self.batch_size = int(self.config['batch_size'])

    def printAlgorConfig(self):
        super(DeepRecommender, self).printAlgorConfig()

    @staticmethod
    def truncated_normal(shape, stddev, device, generator=None):
        import torch
        t = torch.empty(*shape, device=device, dtype=torch.float32)
        return torch.nn.init.trunc_normal_(t, mean=0.0, std=stddev, a=-2 * stddev, b=2 * stddev, generator=generator)

    def initModel(self):
        # the numpy tables are allocated (and np.random advanced) exactly as in the reference,
        # even though the deep models never train them (deepRecommender.py:17)
        super(DeepRecommender, self).initModel()
        import torch
        dev = self._device()
        gen = torch.Generator(device=dev)
        gen.manual_seed(self.engine_seed)      # TF's own RNG stream is not reproducible; ours is
        self.device = dev
        # device tables are `emb_pad` wide: the row kernels move 16-byte slices, so num.factors=50
        # (the shipped confs) is stored as 52 columns with two zero columns that never change
        # (zero gradient -> zero Adam update); exported tables are cut back to emb_size
        self.emb_pad = self.emb_size + (-self.emb_size) % 4
        self.user_embeddings = self.pad_columns(self.truncated_normal((self.num_users, self.emb_size), 0.005, dev, gen))
        self.item_embeddings = self.pad_columns(self.truncated_normal((self.num_items, self.emb_size), 0.005, dev, gen))

    def pad_columns(self, t):
        import torch
        if t.shape[1] == self.emb_pad:
            return t.contiguous()
        out = torch.zeros(t.shape[0], self.emb_pad, device=t.device, dtype=t.dtype)
        out[:, :t.shape[1]] = t
        return out

    # ------------------------------------------------------------------ samplers
    def _mt(self):
        from ..engine import MT19937
        mt = MT19937()
        mt.setstate(random.getstate())
        return mt

    def next_batch_pairwise(self):
        """shuffle(trainingData); batches of `batch_size` rows (last one short); per row one
        negative = choice(item_list) until not rated by the user (deepRecommender.py:29-52)."""
        self.shuffle_training_data()
        csr = self.data.rated_csr()
        u_all, i_all, _ = self.data.training_ids()
        for b in range(0, self.train_size, self.batch_size):
            u = u_all[b:b + self.batch_size]
            i = i_all[b:b + self.batch_size]
            mt = self._mt()
            j = mt.sample_pairwise(csr, u)
            random.setstate(mt.getstate())
            yield u, i, j

    def next_batch_pointwise(self):
        """No shuffle; per interaction (u,i,1) followed by 4 x (u, randint(0,I-1) until unrated, 0)
        (deepRecommender.py:54-77)."""
        csr = self.data.rated_csr()
        u_all, i_all, _ = self.data.training_ids()
        for b in range(0, self.train_size, self.batch_size):
            mt = self._mt()
            out = mt.sample_pointwise(csr, u_all[b:b + self.batch_size], i_all[b:b + self.batch_size])
            random.setstate(mt.getstate())
            yield out
