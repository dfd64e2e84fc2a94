"""BPRMF_batch on the H100 behind the reference's model surface.

Mirrors elliot/recommender/latent_factor_models/BPRMF_batch/BPRMF_batch.py:22-120 (params
`factors, lr, l_w, l_b`, name "BPRNN", batch semantics: batch_size < 1 -> one batch per epoch,
loss accumulation, blockwise get_recommendations) and BPRMF_batch_model.py:15-88 (GlorotUniform
tables, Bi zeros, Adam, `Bi + Gu[s:e] @ Gi^T`, masked top-k with lower-index tie rule).

Exact-stream parity with TensorFlow is impossible here (TF's initializer stream and kernels are
not available): the sampler replays the reference's MT19937 stream bit-exactly, the arithmetic is
checked against the fp64 restatement in oracle/tf_models.py (parity unpinned, see there).
"""
import math
import pickle

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger


class BPRMFBatchModel:
    def __init__(self, factors, learning_rate, l_w, l_b, num_users, num_items, random_seed, device):
        self._factors, self._learning_rate, self._l_w, self._l_b = factors, learning_rate, l_w, l_b
        self._num_users, self._num_items = num_users, num_items
        self.device = torch.device(device)
        self.ld = ops.padded_dim(factors)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))
        lim_u, lim_i = math.sqrt(6.0 / (num_users + factors)), math.sqrt(6.0 / (num_items + factors))

        def table(n, lim):                      # GlorotUniform, BPRMF_batch_model.py:39-42
            t = torch.zeros((n, self.ld), device=self.device)
            t[:, :factors] = (torch.rand((n, factors), device=self.device, generator=g) * 2 - 1) * lim
            return t
        self.Gu, self.Gi = table(num_users, lim_u), table(num_items, lim_i)
        nb = (num_items + 3) // 4 * 4
        self.Bi = torch.zeros(nb, device=self.device)
        z = lambda t: torch.zeros_like(t)
        self.grad = {"Gu": z(self.Gu), "Gi": z(self.Gi), "Bi": z(self.Bi)}
        self.m = {"Gu": z(self.Gu), "Gi": z(self.Gi), "Bi": z(self.Bi)}
        self.v = {"Gu": z(self.Gu), "Gi": z(self.Gi), "Bi": z(self.Bi)}
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)

    def train_step(self, batch):
        """batch = (user, pos, neg) int32 device tensors; returns the batch loss (python float)."""
        tu, ti, tj = batch
        self._loss.zero_()
        ops.bpr_batch_grad_f32(self.Gu, self.Gi, self.Bi, self.grad["Gu"], self.grad["Gi"], self.grad["Bi"], self._factors,
                               tu, ti, tj, self._l_w, self._l_b, loss=self._loss)
        self.step += 1
        for name, var in (("Bi", self.Bi), ("Gu", self.Gu), ("Gi", self.Gi)):     # order of BPRMF_batch_model.py:77-78
            ops.adam_dense_f32(var, self.m[name], self.v[name], self.grad[name], self._learning_rate, self.step)
        return self._loss

    def topk(self, k, mask_indptr, mask_indices, tensor_cores=True):
        bias = self.Bi[:self._num_items]
        if tensor_cores and k <= 16:
            idx, val, _ = ops.score_topk_tc(self.Gu, self.Gi, bias, self._factors, k, mask_indptr, mask_indices, stats=False)
            return idx, val
        return ops.score_topk(self.Gu, self.Gi, bias, self._factors, k, mask_indptr, mask_indices)

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
        self.step = s.get("step", 0)
        for k in self.m:
            if "m" in s: self.m[k].copy_(torch.from_numpy(s["m"][k])); self.v[k].copy_(torch.from_numpy(s["v"][k]))

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))


class BPRMF_batch(RecMixin, BaseRecommenderModel):
    r"""Batch BPR-MF (Adam).  YAML keys as in the reference (BPRMF_batch.py:37-48):
    `epochs, batch_size, factors, lr, l_w, l_b`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "factors", 10, int, None),
            ("_learning_rate", "lr", "lr", 0.001, float, None),
            ("_l_w", "l_w", "l_w", 0.1, float, None),
            ("_l_b", "l_b", "l_b", 0.001, float, None),
        ]
        self.autoset_params()
        if self._batch_size < 1:
            self._batch_size = self._data.transactions                 # BPRMF_batch.py:74-75
        if not torch.cuda.is_available():
            raise RuntimeError("elliot_b200.BPRMF_batch needs a CUDA device (there is no CPU fallback)")
        self._device = torch.device(getattr(self._params, "b200_device", "cuda:0"))
        self._indptr, self._set_idx, self._sorted_idx = train_csr_of(self._data, self._device)
        self._sampler = ops.MtSampler(self._num_users, self._num_items, self._indptr, self._set_idx, self._sorted_idx, seed=42)
        self._model = BPRMFBatchModel(self._factors, self._learning_rate, self._l_w, self._l_b, self._num_users,
                                      self._num_items, self._seed, self._device)

    @property
    def name(self):
        return "BPRNN" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

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
        recs_val, recs_test = self.process_protocol(k)
        return dict(recs_val), dict(recs_test)

    def get_recommendations_tensors(self, k):
        return self._model.topk(k, self._indptr, self._sorted_idx)

    def get_single_recommendation(self, mask, k, *args):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        idx, val = self.get_recommendations_tensors(k)
        idx, val = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
        items = np.array(self._data.items, dtype=object)
        out = {}
        for pu, u in enumerate(self._data.users):
            ok = idx[pu] >= 0
            out[u] = list(zip(items[idx[pu][ok]].tolist(), val[pu][ok].tolist()))
        return out
