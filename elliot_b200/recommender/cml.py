"""CML, collaborative metric learning (Hsieh et al., WWW 2017), on the H100 behind the reference's model surface.

Mirrors elliot/recommender/latent_factor_models/CML/CML.py:55-125 (params `factors, lr, l_w, l_b, margin`, name "CML",
batch_size < 1 -> `transactions`, per-batch losses summed) and CML_model.py:18-135: Gu, Gi and Bi are all Keras
'uniform' embeddings (RandomUniform(-0.05, 0.05), the bias too), Keras Adam over the three tables, and the loss of
train_step as its (B, 1) distances and (B,) biases broadcast it: a B x B hinge, counted by csrc/cml.cu (see there) in
O(B log B) instead of formed.  `censor` is defined there and never called, so nothing clips the rows here either.

Scores are predict's Bi - |Gu - Gi|^2 expanded as (2 Gu).Gi + (Bi - |Gi|^2) - |Gu|^2: the dot-product scorers rank
(2 Gu, Gi, Bi - |Gi|^2) (a per-user constant changes no ranking) and -|Gu|^2 is added to the kept values.  The ranking
rounds as the scorer's bound (oracle/topk_bound.py) with the item offsets as the bias, plus the fp32 rounding of the
offsets themselves (oracle/cml.py::expansion_bound).

Exact-stream parity with TensorFlow is impossible here (TF's initializer stream and kernels are not available): the sampler
replays the reference's MT19937 stream bit-exactly, the arithmetic is checked against the fp64 restatements in
oracle/cml.py (parity unpinned).
"""
import pickle

import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, cuda_device


class CMLModel:
    def __init__(self, factors, learning_rate, l_w, l_b, margin, num_users, num_items, random_seed, device):
        if factors < 2:
            raise ValueError(f"CML needs factors >= 2 (got {factors}): at 1 the reference's tf.squeeze also drops the "
                             "factor axis, which is a different model")
        self._factors, self._learning_rate, self._l_w, self._l_b, self._margin = factors, learning_rate, l_w, l_b, margin
        self._num_users, self._num_items = num_users, num_items
        self.device = torch.device(device)
        self.ld = ops.padded_dim(factors)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))

        def uniform(rows, cols, shape):          # keras 'uniform' = RandomUniform(-0.05, 0.05), CML_model.py:128-135
            t = torch.zeros(shape, device=self.device)
            t.view(shape[0], -1)[:rows, :cols] = torch.rand((rows, cols), device=self.device, generator=g) * 0.1 - 0.05
            return t
        self.Gu = uniform(num_users, factors, (num_users, self.ld))
        self.Gi = uniform(num_items, factors, (num_items, self.ld))
        self.Bi = torch.zeros((num_items + 3) // 4 * 4, device=self.device)        # padded for the vector Adam
        self.Bi[:num_items] = uniform(num_items, 1, (num_items, 1)).view(-1)
        z = lambda t: torch.zeros_like(t)
        self.grad = {"Gu": z(self.Gu), "Gi": z(self.Gi), "Bi": z(self.Bi)}
        self.m = {"Gu": z(self.Gu), "Gi": z(self.Gi), "Bi": z(self.Bi)}
        self.v = {"Gu": z(self.Gu), "Gi": z(self.Gi), "Bi": z(self.Bi)}
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)

    def grads(self, batch, terms=None):
        """Set self._loss to the batch loss and add its gradients to self.grad; terms: see ops.cml_grad_f32."""
        tu, ti, tj = batch
        self._loss.zero_()
        ops.cml_grad_f32(self.Gu, self.Gi, self.Bi, self.grad["Gu"], self.grad["Gi"], self.grad["Bi"], self._factors, tu, ti,
                         tj, self._l_w, self._l_b, self._margin, loss=self._loss, terms=terms)

    def adam(self):
        """One Keras Adam step on the three tables; clears self.grad."""
        self.step += 1
        for name, var in (("Gu", self.Gu), ("Gi", self.Gi), ("Bi", self.Bi)):      # trainable_variables order
            ops.adam_dense_f32(var, self.m[name], self.v[name], self.grad[name], self._learning_rate, self.step)

    def train_step(self, batch):
        """batch = (user, pos, neg) int32 device tensors; returns the batch loss (fp64 device tensor)."""
        self.grads(batch)
        self.adam()
        return self._loss

    def score_operands(self):
        """(2 Gu, Bi - |Gi|^2, -|Gu|^2)"""
        return ops.cml_score_operands_f32(self.Gu, self.Gi, self.Bi, self._num_users, self._num_items)

    def topk(self, k, mask_indptr, mask_indices, tensor_cores=True):
        """masked top-k of Bi - |Gu - Gi|^2 for all users (predict / get_top_k, CML_model.py:101-111)."""
        U2, item_off, user_off = self.score_operands()
        if tensor_cores and k <= 16:
            idx, val, _ = ops.score_topk_tc(U2, self.Gi, item_off, self._factors, k, mask_indptr, mask_indices, stats=False)
        else:
            idx, val = ops.score_topk(U2, self.Gi, item_off, self._factors, k, mask_indptr, mask_indices)
        return idx, ops.add_row_offset_(val, user_off)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from, without the per-user -|Gu|^2."""
        U2, item_off, _ = self.score_operands()
        return ops.score_rank(U2, self.Gi, item_off, self._factors, rel_indptr, rel_items, mask_indptr, mask_indices)

    def get_model_state(self):
        F = self._factors
        return {"Bi": self.Bi[:self._num_items].cpu().numpy(), "Gu": self.Gu[:, :F].cpu().numpy(),
                "Gi": self.Gi[:, :F].cpu().numpy(), "step": self.step,
                "m": {k: t.cpu().numpy() for k, t in self.m.items()}, "v": {k: t.cpu().numpy() for k, t in self.v.items()}}

    def set_model_state(self, s):
        F = self._factors
        self.Bi.zero_(); self.Bi[:self._num_items] = torch.from_numpy(s["Bi"]).to(self.device)
        self.Gu.zero_(); self.Gu[:, :F] = torch.from_numpy(s["Gu"]).to(self.device)
        self.Gi.zero_(); self.Gi[:, :F] = torch.from_numpy(s["Gi"]).to(self.device)
        self.step = s["step"]
        for k in self.m:
            self.m[k].copy_(torch.from_numpy(s["m"][k])); self.v[k].copy_(torch.from_numpy(s["v"][k]))

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))


class CML(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    r"""Collaborative Metric Learning (https://www.cs.cornell.edu/~ylongqi/paper/HsiehYCLBE17.pdf).  YAML keys as in the
    reference (CML.py:66-72): `epochs, batch_size, factors, lr, l_w, l_b, margin`; optional keys `b200_eval` and
    `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "factors", 100, int, None),
            ("_learning_rate", "lr", "lr", 0.001, float, None),
            ("_l_w", "l_w", "l_w", 0.001, float, None),
            ("_l_b", "l_b", "l_b", 0.001, float, None),
            ("_margin", "margin", "margin", 0.5, float, None),
        ]
        self.autoset_params()
        if self._batch_size < 1:
            self._batch_size = self._data.transactions                 # CML.py:78-79
        self._device = cuda_device(self._params, "CML")
        self._indptr, self._set_idx, self._sorted_idx = train_csr_of(self._data, self._device)
        self._sampler = ops.MtSampler(self._num_users, self._num_items, self._indptr, self._set_idx, self._sorted_idx, seed=42)
        self._model = CMLModel(self._factors, self._learning_rate, self._l_w, self._l_b, self._margin, self._num_users,
                               self._num_items, self._seed, self._device)

    @property
    def name(self):
        return "CML" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        T = self._data.transactions
        for it in self.iterate(self._epochs):
            loss = 0.0
            tu, ti, tj = self._sampler.step(T)                           # same triples as the reference's Sampler.step
            for s in range(0, T, self._batch_size):
                e = min(s + self._batch_size, T)
                loss += float(self._model.train_step((tu[s:e].contiguous(), ti[s:e].contiguous(), tj[s:e].contiguous())).item())
            self.evaluate(it, loss / (it + 1))

    def get_recommendations(self, k: int = 100):
        return super().get_recommendations(k)
