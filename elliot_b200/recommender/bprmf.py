"""BPRMF on the H100 behind the reference's model surface.

Mirrors elliot/recommender/latent_factor_models/BPRMF/BPRMF.py:23-129 (constructor contract,
`_params_list` keys/defaults, name, train(), get_recommendations()) and BPRMF_model.py:14-139
(MFModel: init stream, state dict, pickle weights).  All arithmetic of the hot path runs in
the CUDA kernels behind include/elliot_b200.h:

  mode "exact" (default)  — the reference's own semantics: one legacy-MT19937 stream of
      (u,i,j) triples replayed on the device (eb_mt_sampler_step), strictly sequential fp64
      SGD reproduced by row turn counters (eb_bpr_exact_f64), fp64 scoring + top-k.  Same
      splits + seeds => same tables (<=1e-12), same top-k lists, same nDCG.
  mode "hogwild"          — throughput mode: fused Philox sampling + fp32 Hogwild step
      (eb_bpr_step_sampled_f32).  Same distribution, different stream; reports its own nDCG.

Extra YAML keys (absent from the reference, all optional): `b200_mode`, `b200_batch`, `b200_eval`
(`device`: metrics computed by `eb_eval_topk_f64` from the top-k tensor; `host`: the reference's dict path; default
`host` in exact mode, `device` in hogwild mode).
"""
import pickle

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, cuda_device


class MFModel:
    """Device-resident factor model with the reference MFModel's interface subset
    (BPRMF_model.py:14-139): same init stream, same state-dict keys, pickle weights."""

    def __init__(self, F, data, lr, user_regularization, bias_regularization, positive_item_regularization,
                 negative_item_regularization, random_seed, mode="exact", device="cuda:0"):
        np.random.seed(random_seed)                                   # BPRMF_model.py:24
        self._factors, self._data, self._mode = F, data, mode
        self._learning_rate = lr
        self._user_regularization, self._bias_regularization = user_regularization, bias_regularization
        self._positive_item_regularization = positive_item_regularization
        self._negative_item_regularization = negative_item_regularization
        self.device = torch.device(device)
        nu, ni = len(data.users), len(data.items)
        # BPRMF_model.py:49-56: biases zero, U ~ N(0, .1) drawn first, then V, legacy global stream
        U0 = np.random.normal(loc=0, scale=0.1, size=(nu, F))
        V0 = np.random.normal(loc=0, scale=0.1, size=(ni, F))
        self._user_bias = np.zeros(nu)                                 # never used by predictions (BPRMF_model.py:62-68)
        self._set_tables(U0, V0, np.zeros(ni))

    def _set_tables(self, U, V, b):
        F = self._factors
        if self._mode == "exact":
            self.ld = F
            self.U = torch.from_numpy(np.ascontiguousarray(U, np.float64)).to(self.device)
            self.V = torch.from_numpy(np.ascontiguousarray(V, np.float64)).to(self.device)
            self.b = torch.from_numpy(np.ascontiguousarray(b, np.float64)).to(self.device)
        else:
            self.ld = ops.padded_dim(F)
            self.U = torch.zeros((U.shape[0], self.ld), dtype=torch.float32, device=self.device)
            self.V = torch.zeros((V.shape[0], self.ld), dtype=torch.float32, device=self.device)
            self.U[:, :F] = torch.from_numpy(U).to(self.device, torch.float32)
            self.V[:, :F] = torch.from_numpy(V).to(self.device, torch.float32)
            self.b = torch.from_numpy(b).to(self.device, torch.float32)

    @property
    def name(self):
        return "MF"

    def hyper(self):
        return (self._learning_rate, self._user_regularization, self._bias_regularization,
                self._positive_item_regularization, self._negative_item_regularization)

    # ---- training (BPRMF_model.py:87-117) ------------------------------------------------
    def train_step(self, batch, loss=None):
        """batch = (u, i, j) int32 device tensors of any length, applied in order."""
        tu, ti, tj = batch
        if self._mode == "exact":
            ops.bpr_exact_f64(self.U, self.V, self.b, self._factors, tu, ti, tj, *self.hyper(), loss=loss)
        else:
            ops.bpr_step_f32(self.U, self.V, self.b, self._factors, tu, ti, tj, *self.hyper(), loss=loss)

    # ---- scoring (BPRMF_model.py:70-85) ----------------------------------------------------
    def topk(self, k, mask_indptr, mask_indices, users=None):
        if self._mode != "exact" and users is None and k <= 16:          # fp32 tables: tensor-core path, same result
            idx, val, _ = ops.score_topk_tc(self.U, self.V, self.b, self._factors, k, mask_indptr, mask_indices, stats=False)
            return idx, val
        return ops.score_topk(self.U, self.V, self.b, self._factors, k, mask_indptr, mask_indices, users=users)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        return ops.score_rank(self.U, self.V, self.b, self._factors, rel_indptr, rel_items, mask_indptr, mask_indices)

    # ---- state (BPRMF_model.py:119-139) ----------------------------------------------------
    def get_model_state(self):
        F = self._factors
        return {"_user_bias": self._user_bias,
                "_item_bias": self.b.double().cpu().numpy(),
                "_user_factors": self.U[:, :F].double().cpu().numpy(),
                "_item_factors": self.V[:, :F].double().cpu().numpy()}

    def set_model_state(self, s):
        self._user_bias = s["_user_bias"]
        self._set_tables(s["_user_factors"], s["_item_factors"], s["_item_bias"])

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)


class BPRMF(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    r"""Bayesian Personalized Ranking MF (https://arxiv.org/abs/1205.2618) on the H100.

    YAML block identical to the reference's (BPRMF.py:37-56):
        BPRMF: {meta: {...}, epochs, factors, lr, bias_regularization, user_regularization,
                positive_item_regularization, negative_item_regularization, ...}
    """

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "f", 10, int, None),
            ("_learning_rate", "lr", "lr", 0.05, None, None),
            ("_bias_regularization", "bias_regularization", "bias_reg", 0, None, None),
            ("_user_regularization", "user_regularization", "u_reg", 0.0025, None, None),
            ("_positive_item_regularization", "positive_item_regularization", "pos_i_reg", 0.0025, None, None),
            ("_negative_item_regularization", "negative_item_regularization", "neg_i_reg", 0.00025, None, None),
            ("_update_negative_item_factors", "update_negative_item_factors", "up_neg_i_f", True, None, None),
            ("_update_users", "update_users", "up_u", True, None, None),
            ("_update_items", "update_items", "up_i", True, None, None),
            ("_update_bias", "update_bias", "up_b", True, None, None),
        ]
        self.autoset_params()
        self._mode = getattr(self._params, "b200_mode", "exact")
        if self._mode not in ("exact", "hogwild"):
            raise Exception("b200_mode must be 'exact' or 'hogwild'")
        self._hog_batch = int(getattr(self._params, "b200_batch", 1 << 20))
        if self._mode == "hogwild" and not hasattr(self._params, "b200_eval"):
            self._params.b200_eval = "device"          # throughput mode: metrics straight from the top-k tensor
        self._batch_size = 1                                    # BPRMF.py:80 (YAML batch_size ignored)
        self._device = cuda_device(self._params, "BPRMF")
        # construction order as in BPRMF.py:83-91: model (seeds np.random with the model seed),
        # then the sampler (reseeds the global stream with 42)
        self._model = MFModel(self._factors, self._data, self._learning_rate, self._user_regularization,
                              self._bias_regularization, self._positive_item_regularization,
                              self._negative_item_regularization, self._seed, mode=self._mode, device=self._device)
        self._indptr, self._set_idx, self._sorted_idx = train_csr_of(self._data, self._device)
        self._sampler = ops.MtSampler(self._num_users, self._num_items, self._indptr, self._set_idx,
                                      self._sorted_idx, seed=42)     # custom_sampler.py:15
        np.random.seed(42)                                      # keep the host's global stream where the reference leaves it
        self._hog_counter = 0
        self._loss_dev = torch.zeros(1, dtype=torch.float64, device=self._device)
        # per-user membership signatures shorten the sampler's load chain on large catalogues and cost time on small,
        # L2-resident ones; the samples are identical either way
        self._filter = ops.bloom_build(self._indptr, self._sorted_idx, self._num_users) \
            if self._mode == "hogwild" and self._num_items >= 500_000 else None

    @property
    def name(self):
        return "BPRMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    # ---- training (BPRMF.py:113-129) -------------------------------------------------------
    def train(self):
        if self._restore:
            return self.restore_weights()
        T = self._data.transactions
        for it in self.iterate(self._epochs):
            self._loss_dev.zero_()
            if self._mode == "exact":
                batch = self._sampler.step(T)                    # one continuous MT19937(42) stream across epochs
                self._model.train_step(batch, loss=self._loss_dev)
            else:
                done = 0
                while done < T:
                    n = min(self._hog_batch, T - done)
                    ops.bpr_step_sampled_f32(self._model.U, self._model.V, self._model.b, self._factors,
                                             self._num_users, self._num_items, self._indptr, self._sorted_idx, n,
                                             self._seed, self._hog_counter, *self._model.hyper(), loss=self._loss_dev,
                                             filter=self._filter)
                    self._hog_counter += n
                    done += n
            self.evaluate(it, float(self._loss_dev.item()))
