"""LMF, the reference's logistic matrix factorization (latent_factor_models/LogisticMF/, YAML key `LMF`), on the H100
behind the reference's model surface.

Mirrors logistic_matrix_factorization.py + logistic_matrix_factorization_model.py: x = g_u . g_i + b_u + b_i with
GlorotUniform Gu / Gi and zero Bu / Bi; per batch the loss is the SUM over the samples of -(alpha y x - (1 + alpha y)
log(1 + e^x)) plus reg (|g_u|^2 / 2 + |g_i|^2 / 2) over the looked-up rows; Keras Adagrad (initial accumulator 0.1,
epsilon 1e-7).  Each epoch runs two passes of `transactions` samples from one continuing pointwise pos/neg stream, and
BOTH update Gi and Bi only: the reference's `set_update_user` assigns a Python attribute inside a tf.function, which
happens only while tracing, and `train_step`'s `if self._user_update:` was frozen to the item branch when the first
(item) pass traced it, for both batch shapes; the "user" pass reuses those graphs (DESIGN §4.20).  Gu and Bu therefore
keep their initial values; the loss still carries the g_u regulariser.

Per batch: ONE fused kernel (eb_pointwise_mf_step_f32, LMF) scatters dGi / dBi and adds the loss, then
eb_adagrad_rows_f32 applies TF's sparse Adagrad to the item rows the batch touched, once each, and clears their
gradients: TF leaves untouched rows and their accumulators alone, so this is exact.  softplus and sigmoid are computed in
overflow-free forms (the reference's log(1 + exp(x)) is inf above x ~ 88.7 in fp32; DESIGN §5).  Recommendations are
b_u + b_i + g_u . g_i: the scorers rank g_u . g_i + b_i and b_u is added to the kept values.  TensorFlow parity is
UNPINNED (checker: oracle/pointwise_mf.py).
"""
import math
import pickle

import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import PairScoreRecs, RankRecs, TopKRecs, cuda_device

ADAGRAD_INIT, ADAGRAD_EPS = 0.1, 1e-7                                    # tf.keras.optimizers.Adagrad defaults


class LMFModel:
    """Gu, Gi [n, ld] (factor columns padded to a multiple of 4 with zeros), Bu, Bi, the Adagrad accumulators of Gi and
    Bi, their gradient tables and the per-item step stamps of eb_adagrad_rows_f32."""

    def __init__(self, num_users, num_items, factors, reg, alpha, learning_rate, random_seed, device):
        assert 2 <= factors <= 128
        self.nu, self.ni, self.f, self.reg, self.alpha, self.lr = num_users, num_items, factors, reg, alpha, learning_rate
        self.fp = (factors + 3) // 4 * 4
        self.ld = ops.padded_dim(self.fp)
        self.device = torch.device(device)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))

        def glorot(rows):                                                # tf.initializers.GlorotUniform on [rows, factors]
            t = torch.zeros((rows, self.ld), device=self.device)
            lim = math.sqrt(6.0 / (rows + factors))
            t[:, :factors] = (torch.rand((rows, factors), device=self.device, generator=g) * 2 - 1) * lim
            return t
        self.P = {"Gu": glorot(num_users), "Gi": glorot(num_items),
                  "Bu": torch.zeros(num_users, device=self.device), "Bi": torch.zeros(num_items, device=self.device)}
        self.acc = {"Gi": torch.full_like(self.P["Gi"], ADAGRAD_INIT), "Bi": torch.full_like(self.P["Bi"], ADAGRAD_INIT)}
        self.G = {"Gi": torch.zeros_like(self.P["Gi"]), "Bi": torch.zeros_like(self.P["Bi"])}
        self.stamp = torch.zeros(num_items, dtype=torch.int64, device=self.device)
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)

    def grads(self, batch):
        """Add the batch's item-side gradients to self.G and its loss to self._loss."""
        u, it, y = batch
        P = self.P
        ops.pointwise_mf_step_f32(P["Gu"], P["Gi"], self.fp, u, it, y, self.G["Gi"], ops.LMF_LOGPOST, bu=P["Bu"], bi=P["Bi"],
                                  dbi=self.G["Bi"], alpha=self.alpha, lam=self.reg, loss=self._loss)

    def adagrad(self, it):
        """TF's sparse Adagrad on the item rows `it` touched (and their biases); clears their gradients."""
        self.step += 1
        ops.adagrad_rows_f32(self.P["Gi"], self.acc["Gi"], self.G["Gi"], it, self.stamp, self.step, self.lr, width=self.f,
                             bvar=self.P["Bi"], bacc=self.acc["Bi"], bgrad=self.G["Bi"], eps=ADAGRAD_EPS)

    def train_step(self, batch):
        """batch = (user int32, item int32, label float32) device tensors; returns the batch loss tensor (device)."""
        self._loss.zero_()
        self.grads(batch)
        self.adagrad(batch[1])
        return self._loss

    def topk(self, k, mask_indptr, mask_indices):
        """masked top-k of b_u + b_i + g_u . g_i for all users (predict_batch / get_top_k)."""
        if k <= 16:
            idx, val, _ = ops.score_topk_tc(self.P["Gu"], self.P["Gi"], self.P["Bi"], self.f, k, mask_indptr, mask_indices,
                                            stats=False)
        else:
            idx, val = ops.score_topk(self.P["Gu"], self.P["Gi"], self.P["Bi"], self.f, k, mask_indptr, mask_indices)
        return idx, ops.add_row_offset_(val, self.P["Bu"])

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from, without b_u (a per-user constant)."""
        return ops.score_rank(self.P["Gu"], self.P["Gi"], self.P["Bi"], self.f, rel_indptr, rel_items, mask_indptr, mask_indices)

    def pair_scores(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """Each relevant entry's score in the user's full list (-inf for a train item, NaN outside the catalogue)."""
        return ops.score_pairs_f32(self.P["Gu"], self.P["Gi"], self.fp, rel_indptr, rel_items, item_bias=self.P["Bi"],
                                   user_off=self.P["Bu"], mask_indptr=mask_indptr, mask_indices=mask_indices)

    def get_model_state(self):
        cpu = lambda d: {k: v.cpu().numpy() for k, v in d.items()}
        return {"P": cpu(self.P), "acc": cpu(self.acc), "stamp": self.stamp.cpu().numpy(), "step": self.step}

    def set_model_state(self, s):
        for k in self.P:
            self.P[k].copy_(torch.from_numpy(s["P"][k]))
        for k in self.acc:
            self.acc[k].copy_(torch.from_numpy(s["acc"][k]))
        self.stamp.copy_(torch.from_numpy(s["stamp"]))
        self.step = s["step"]

    def save_weights(self, path):
        with open(path, "wb") as fh:
            pickle.dump(self.get_model_state(), fh)

    def load_weights(self, path):
        with open(path, "rb") as fh:
            self.set_model_state(pickle.load(fh))


class LMF(TopKRecs, RankRecs, PairScoreRecs, RecMixin, BaseRecommenderModel):
    r"""Logistic Matrix Factorization (https://web.stanford.edu/~rezab/nips2014workshop/submits/logmat.pdf).  YAML keys
    as in the reference (lr, factors, reg, alpha); optional keys `b200_eval` and `b200_device`.  `factors` must be in
    [2, 128]: at 1 the reference's tf.squeeze drops the factor axis and sums the dot over the whole batch, a different
    model."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_learning_rate", "lr", "lr", 0.001, None, None),
            ("_factors", "factors", "factors", 10, None, None),
            ("_l_w", "reg", "reg", 0.1, None, None),
            ("_alpha", "alpha", "alpha", 0.5, None, None),
        ]
        self.autoset_params()
        f = int(self._factors)
        if f == 1:
            raise ValueError("LMF: factors=1 is refused: the reference's tf.squeeze then drops the factor axis and "
                             "reduce_sum adds g_u * g_i over the whole batch, a different model")
        if not 1 <= f <= 128:
            raise ValueError(f"LMF: factors={self._factors} is outside [1, 128], the widths the step and scoring kernels take")
        if self._batch_size < 1:
            self._batch_size = self._data.transactions
        self._device = cuda_device(self._params, "LMF")
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._filter = ops.bloom_build(self._indptr, self._sorted_idx, self._num_users)
        self._model = LMFModel(self._num_users, self._num_items, f, float(self._l_w), float(self._alpha),
                               float(self._learning_rate), self._seed, self._device)
        self._drawn = 0

    @property
    def name(self):
        return "LMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def _samples(self, T):
        u, i, y = ops.pointwise_sample_philox(self._num_users, self._num_items, self._indptr, self._sorted_idx, T, 42,
                                              first=self._drawn, filter=self._filter)
        self._drawn += T
        return u, i, y

    def train(self):
        if self._restore:
            return self.restore_weights()
        T = self._data.transactions
        for it in self.iterate(self._epochs):
            loss = 0.0
            for _ in range(2):                                           # the "item" pass, then the "user" pass: both item steps
                u, i, y = self._samples(T)
                for s in range(0, T, self._batch_size):
                    e = min(s + self._batch_size, T)
                    loss += float(self._model.train_step((u[s:e], i[s:e], y[s:e])).item())
            self.evaluate(it, loss / (it + 1))
