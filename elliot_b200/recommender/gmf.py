"""GMF (Generalized Matrix Factorization, NeuMF's MF branch) on the H100 behind the reference's model surface
(SURVEY.md §8f #3).

Mirrors elliot/recommender/neural/GeneralizedMF/generalized_matrix_factorization.py:24-120 (params `lr, mf_factors,
is_edge_weight_train`; name prefix "GeneralizedMF"; `transactions` samples per epoch from the pointwise pos/neg sampler) and
generalized_matrix_factorization_model.py:18-92 for `is_edge_weight_train: True` (the default): out = sigmoid((U[u]*I[i]).h),
BinaryCrossentropy, Keras Adam over the full tables and h.  (`is_edge_weight_train: False` builds an int32 scalar
`tf.Variable(initial_value=1, shape=[f, 1])` in the reference and cannot multiply a float matrix; it is not mirrored.)
One fused kernel per batch does gather -> score -> loss -> gradient scatter (eb_gmf_step_grads); recommendations rank the
plain dot products (U*h).I^T with the tensor-core scoring kernel — sigmoid is monotone — and only the k kept logits are
turned into probabilities.  The sampler draws the reference's distribution from a Philox stream (the reference interleaves
np.random and `random.getrandbits`; that stream is not replayed).  TensorFlow parity is UNPINNED (checker:
oracle/tf_models.py::gmf_forward_backward).  mf_factors is padded to the kernels' row stride; it must be <= 128.
"""
import math
import pickle

import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import cuda_device, recs_dict


class GeneralizedMatrixFactorizationModel:
    def __init__(self, num_users, num_items, embed_mf_size, is_edge_weight_train, learning_rate, random_seed, device):
        if not is_edge_weight_train:
            raise NotImplementedError("is_edge_weight_train: False is not runnable in the reference either (int32 edge weights)")
        assert 1 <= embed_mf_size <= 128
        self.nu, self.ni, self.f, self.lr = num_users, num_items, embed_mf_size, learning_rate
        self.fp = (embed_mf_size + 3) // 4 * 4                          # kernels work on float4 columns; padding stays zero
        self.ld = ops.padded_dim(self.fp)
        self.device = torch.device(device)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))

        def glorot(rows, cols, fan_in, fan_out, ld):                    # GlorotUniform (:34)
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            t = torch.zeros((rows, ld), device=self.device)
            t[:, :cols] = (torch.rand((rows, cols), device=self.device, generator=g) * 2 - 1) * lim
            return t
        f = self.f
        self.P = {"U": glorot(num_users, f, num_users, f, self.ld), "I": glorot(num_items, f, num_items, f, self.ld),
                  "h": glorot(1, f, f, 1, self.ld).reshape(-1).contiguous()}
        z = lambda t: torch.zeros_like(t)
        self.G = {k: z(v) for k, v in self.P.items()}
        self.M = {k: z(v) for k, v in self.P.items()}
        self.V = {k: z(v) for k, v in self.P.items()}
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)

    def train_step(self, batch):
        """batch = (user int32, item int32, label float32) device tensors; returns the batch loss tensor."""
        u, it, y = batch
        P, G = self.P, self.G
        self._loss.zero_()
        ops.gmf_step_grads(P["U"], P["I"], P["h"], self.fp, u, it, y, G["U"], G["I"], G["h"], loss=self._loss)
        self.step += 1
        for k in P:
            ops.adam_dense_f32(P[k], self.M[k], self.V[k], G[k], self.lr, self.step)
        return self._loss

    def get_recs_topk(self, k, mask_indptr, mask_indices):
        """masked top-k of sigmoid((U*h) . I^T) for all users (get_recs/get_top_k, :76-92)."""
        Uh = ops.gmf_scale_rows(self.P["U"], self.P["h"], self.fp)
        if k <= 16:
            idx, val, _ = ops.score_topk_tc(Uh, self.P["I"], None, self.f, k, mask_indptr, mask_indices, stats=False)
        else:
            idx, val = ops.score_topk(Uh, self.P["I"], None, self.f, k, mask_indptr, mask_indices)
        return idx, ops.sigmoid_(val.contiguous())

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists get_recs_topk() selects from: (U*h) . I^T before the sigmoid."""
        Uh = ops.gmf_scale_rows(self.P["U"], self.P["h"], self.fp)
        return ops.score_rank(Uh, self.P["I"], None, self.f, rel_indptr, rel_items, mask_indptr, mask_indices)

    def get_model_state(self):
        return {"P": {k: v.cpu().numpy() for k, v in self.P.items()}, "step": self.step,
                "M": {k: v.cpu().numpy() for k, v in self.M.items()}, "V": {k: v.cpu().numpy() for k, v in self.V.items()}}

    def set_model_state(self, s):
        for k in self.P:
            self.P[k].copy_(torch.from_numpy(s["P"][k])); self.M[k].copy_(torch.from_numpy(s["M"][k])); self.V[k].copy_(torch.from_numpy(s["V"][k]))
        self.step = s["step"]

    def save_weights(self, path):
        with open(path, "wb") as fh:
            pickle.dump(self.get_model_state(), fh)

    def load_weights(self, path):
        with open(path, "rb") as fh:
            self.set_model_state(pickle.load(fh))


class GMF(RecMixin, BaseRecommenderModel):
    r"""Neural Collaborative Filtering, GMF branch (https://arxiv.org/abs/1708.05031).  YAML keys as in the reference."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_learning_rate", "lr", "lr", 0.001, None, None),
            ("_mf_factors", "mf_factors", "mffactors", 10, None, None),
            ("_is_edge_weight_train", "is_edge_weight_train", "isedgeweighttrain", True, None, None),
        ]
        self.autoset_params()
        if self._batch_size < 1:
            self._batch_size = self._data.transactions
        self._device = cuda_device(self._params, "GMF")
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._filter = ops.bloom_build(self._indptr, self._sorted_idx, self._num_users)
        self._model = GeneralizedMatrixFactorizationModel(self._num_users, self._num_items, int(self._mf_factors),
                                                          self._is_edge_weight_train, self._learning_rate, self._seed, self._device)
        self._drawn = 0

    @property
    def name(self):
        return "GeneralizedMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        T = self._data.transactions
        for it in self.iterate(self._epochs):
            loss = 0.0
            u, i, y = ops.pointwise_sample_philox(self._num_users, self._num_items, self._indptr, self._sorted_idx, T, 42,
                                                  first=self._drawn, filter=self._filter)
            self._drawn += T
            for s in range(0, T, self._batch_size):
                e = min(s + self._batch_size, T)
                loss += float(self._model.train_step((u[s:e], i[s:e], y[s:e])).item())
            self.evaluate(it, loss / (it + 1))

    def get_recommendations(self, k: int = 100):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        out = recs_dict(self._data, *self._model.get_recs_topk(k, self._indptr, self._sorted_idx))
        return out, out

    def get_recommendations_tensors(self, k: int = 10):
        return self._model.get_recs_topk(k, self._indptr, self._sorted_idx)

    def get_rank_tensors(self, rel_indptr, rel_items):
        return self._model.rank(rel_indptr, rel_items, self._indptr, self._sorted_idx)
