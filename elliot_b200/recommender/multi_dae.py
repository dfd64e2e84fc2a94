"""MultiDAE on the H100 behind the reference's model surface (SURVEY.md §8f #3: "VAE minus sampling/KL").

Mirrors elliot/recommender/autoencoders/dae/multi_dae.py:24-110 (same YAML keys as MultiVAE, per-epoch shuffled user
batches from sparse_sampler.py:13-25) and multi_dae_model.py:20-145: l2-normalised, dropped-out user row ->
tanh Dense(I -> H) -> tanh Dense(H -> L) = the code -> tanh Dense(L -> H) -> Dense(H -> I); loss = per-user
multinomial negative log-likelihood (mean over the batch), Keras Adam; `reg_lambda` is accepted and inert as in the
reference (regulariser losses are never added, multi_dae_model.py:38-44 vs :118-125).  Built from the MultiVAE
kernels: CSR gather-sum input layer, tensor-core dense layers (eb_gemm_bf16_tn), fused softmax/NLL.  TensorFlow parity
is UNPINNED (TF cannot run here): tests check the gradients against the fp64 restatement oracle/tf_models.py.
"""
import random

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from .multi_vae import VariationalAutoEncoder, epoch_user_order


class DenoisingAutoEncoder(VariationalAutoEncoder):
    """Same containers, optimiser state, bf16 operand copies and data-parallel hook as the VAE model; the code layer
    is one tanh Dense of width L and there is no sampling / KL term."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.native = False                       # launch-by-launch sequence of the tested kernels (below)

    def _code_width(self):
        return self.L

    def _forward(self, rows, step_id, kl_sum=None, train=True):
        B, H, L, I = rows.numel(), self.H, self.L, self.I
        h1 = torch.empty((B, H), device=self.device)
        ops.vae_embed_fwd(self.P["W1"], self.P["b1"], self.indptr, self.indices, rows, h1,
                          self.drop if train else 0.0, self.seed * 7919 + step_id + self._salt)
        zm = ops.gemm_bf16_tn(ops.to_bf16(h1), self.W2b, B, L, H, bias=self.P["b2"], act=1)       # multi_dae_model.py:40-52
        h2 = ops.gemm_bf16_tn(ops.to_bf16(zm), self.W3b, B, H, L, bias=self.P["b3"], act=1)
        logits = ops.gemm_bf16_tn(ops.to_bf16(h2), self.W4b, B, I, H, bias=self.P["b4"])
        return h1, zm, zm, h2, logits

    def compute_grads(self, rows, anneal, sid):
        B, H, L, I = rows.numel(), self.H, self.L, self.I
        h1, zm, _, h2, logits = self._forward(rows, sid)
        ops.vae_softmax(logits, self.indptr, self.indices, rows, nll_sum=self._acc[1:2], write_grad=True)
        dlogits, G = logits, self.G                                                               # in place
        dl_b, h1_b, zm_b, h2_b = ops.to_bf16(dlogits), ops.to_bf16(h1), ops.to_bf16(zm), ops.to_bf16(h2)
        ops.gemm_bf16(dl_b, h2_b, I, H, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W4"]); ops.colsum(dlogits, G["b4"])
        dpre2 = ops.tanh_bwd(ops.gemm_bf16(dl_b, self.W4b, B, H, I, b_rows_are_k=True), h2)
        dpre2_b = ops.to_bf16(dpre2)
        ops.gemm_bf16(dpre2_b, zm_b, H, L, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W3"]); ops.colsum(dpre2, G["b3"])
        dprez = ops.tanh_bwd(ops.gemm_bf16(dpre2_b, self.W3b, B, L, H, b_rows_are_k=True), zm)
        dprez_b = ops.to_bf16(dprez)
        ops.gemm_bf16(dprez_b, h1_b, L, H, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W2"]); ops.colsum(dprez, G["b2"])
        dpre1 = ops.tanh_bwd(ops.gemm_bf16(dprez_b, self.W2b, B, H, L, b_rows_are_k=True), h1)
        ops.colsum(dpre1, G["b1"])
        ops.vae_embed_bwd(G["W1"], self.indptr, self.indices, rows, dpre1, self.drop, self.seed * 7919 + sid + self._salt)


class MultiDAE(RecMixin, BaseRecommenderModel):
    r"""Collaborative denoising autoencoder (https://dl.acm.org/doi/10.1145/3178876.3186150).  YAML keys as in the
    reference (multi_dae.py:36-50)."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        random.seed(42)                                              # sparse_sampler.py:10
        if self._batch_size < 1:
            self._batch_size = self._num_users
        self._params_list = [
            ("_intermediate_dim", "intermediate_dim", "intermediate_dim", 600, None, None),
            ("_latent_dim", "latent_dim", "latent_dim", 200, None, None),
            ("_lambda", "reg_lambda", "reg_lambda", 0.01, None, None),
            ("_learning_rate", "lr", "lr", 0.001, None, None),
            ("_dropout_rate", "dropout_pkeep", "dropout_pkeep", 1, None, None),
        ]
        self.autoset_params()
        self._dropout_rate = 1. - self._dropout_rate
        if not torch.cuda.is_available():
            raise RuntimeError("elliot_b200.MultiDAE needs a CUDA device (there is no CPU fallback)")
        self._device = torch.device(getattr(self._params, "b200_device", "cuda:0"))
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._model = DenoisingAutoEncoder(self._num_items, int(self._intermediate_dim), int(self._latent_dim), self._learning_rate,
                                           self._dropout_rate, self._lambda, self._seed, self._indptr, self._sorted_idx, self._device)

    @property
    def name(self):
        return "MultiDAE" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        for it in self.iterate(self._epochs):
            loss = 0
            order = torch.tensor(epoch_user_order(self._num_users), dtype=torch.int32, device=self._device)
            for s in range(0, self._num_users, self._batch_size):
                loss += self._model.train_step(order[s:s + self._batch_size].contiguous(), 0.0)
            self.evaluate(it, loss / (it + 1))

    def get_recommendations(self, k: int = 100):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        out = {}
        items = np.array(self._data.items, dtype=object)
        for offset in range(0, self._num_users, self._batch_size):              # recommender_utils_mixin.py:63-73
            stop = min(offset + self._batch_size, self._num_users)
            rows = torch.arange(offset, stop, dtype=torch.int32, device=self._device)
            idx, val = self._model.predict_topk(rows, k, self._indptr, self._sorted_idx)
            idx, val = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
            for r, pu in enumerate(range(offset, stop)):
                ok = idx[r] >= 0
                out[self._data.users[pu]] = list(zip(items[idx[r][ok]].tolist(), val[r][ok].tolist()))
        return out, out
