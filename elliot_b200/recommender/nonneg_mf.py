"""NonNegMF (Luo et al. 2014, "An efficient non-negative matrix-factorization-based approach to collaborative filtering
for recommender systems") on the H100.

Mirrors latent_factor_models/NonNegMF/non_negative_matrix_factorization.py (`_params_list` keys and defaults factors
10, lr 0.001, reg 0.1; batch_size < 1 becomes `transactions`, used only in the name; mu = np.mean(sp_i_train_ratings);
train() = one train_step and one evaluation per epoch) and non_negative_matrix_factorization_model.py (P, then Q, drawn
by RandomState(seed).normal; the epoch; predict; the pickled state dict).  The reference allocates its biases and
per-epoch sums with np.empty; this build starts them from zero, the reference's stated intent (DESIGN §5).

One epoch on the device (csrc/nonneg_mf.cu), every rounding as in the reference:
  eb_nnmf_dots_f64        dot_k = Q[i].P[u] for every rating of the dict-order CSR (slope_one.dict_order_csr);
  eb_nnmf_bias_chain_f64  est_k and the bu / bi updates, one thread walking the ratings in order;
  eb_nnmf_row_update_f64  Q from the item-major CSC (ascending users, each entry's rating position) into a second
                          buffer, then P in place from the CSR: both read the start-of-epoch tables.
Scores are eb_score_topk_f64's P[u].Q[i] + bi[i], then + bu[u], then + mu, in the reference's order of additions.
`meta.save_weights` / `meta.restore` use the reference's pickle dict; evaluation-time negative sampling raises
NotImplementedError.
"""
import pickle

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, check_free, cuda_device, upload
from .slope_one import dict_order_csr


class NonNegMFModel:
    """The device tables and the epoch, with the reference NonNegMFModel's constructor and state dict."""

    def __init__(self, data, num_users, num_items, global_mean, embed_mf_size, lambda_weights, learning_rate=0.01,
                 random_seed=42, device="cuda:0"):
        self.device = torch.device(device)
        self.n_users, self.n_items, self.F = num_users, num_items, int(embed_mf_size)
        self._mu, self._reg, self._lr = global_mean, lambda_weights, learning_rate
        indptr, items, ratings = dict_order_csr(data)
        self.nnz = int(indptr[-1])
        check_free("NonNegMF", self.device, *self.working_set())
        rs = np.random.RandomState(random_seed)
        P = rs.normal(size=(num_users, self.F))
        Q = rs.normal(size=(num_items, self.F))
        self.set_model_state({"_user_bias": np.zeros(num_users), "_item_bias": np.zeros(num_items),
                              "_user_embeddings": P, "_item_embeddings": Q})
        self.Q2 = torch.empty_like(self.Q)
        self.indptr, self.items = upload(indptr, self.device, torch.int64), upload(items, self.device, torch.int32)
        self.ratings = upload(ratings, self.device, torch.float64)
        # the item-major view: a stable sort by item keeps every item's ratings in ascending user order
        pos = np.argsort(items, kind="stable")
        c_indptr = np.zeros(num_items + 1, np.int64)
        np.cumsum(np.bincount(items, minlength=num_items), out=c_indptr[1:])
        users = np.repeat(np.arange(num_users, dtype=np.int32), np.diff(indptr))
        self.c_indptr, self.c_users = upload(c_indptr, self.device, torch.int64), upload(users[pos], self.device, torch.int32)
        self.c_pos = upload(pos, self.device, torch.int64)
        self.dots = torch.empty(self.nnz, dtype=torch.float64, device=self.device)
        self.est = torch.empty_like(self.dots)

    def working_set(self):
        """(bytes on the device, a description)."""
        g = 2 ** 30
        tables = ((self.n_users + 2 * self.n_items) * self.F + self.n_users + self.n_items) * 8
        csr = 2 * self.nnz * 12 + (self.n_users + self.n_items + 2) * 8 + self.nnz * 8
        per_rating = 2 * self.nnz * 8
        return tables + csr + per_rating, (f"P, Q, a second Q and the biases {tables / g:.2f} GiB, the CSR, the CSC and the "
                                           f"ratings {csr / g:.2f} GiB, dot and est per rating {per_rating / g:.2f} GiB")

    def train_step(self, mark=None):
        """One epoch.  `mark(phase)`, when given, is called as each phase has been queued (dots, chain, items, users)."""
        mark = mark or (lambda phase: None)
        ops.nnmf_dots_f64(self.P, self.Q, self.indptr, self.items, out=self.dots)
        mark("dots")
        ops.nnmf_bias_chain_f64(self.indptr, self.items, self.ratings, self.dots, self._mu, self._lr, self._reg, self.bu,
                                self.bi, out=self.est)
        mark("chain")
        ops.nnmf_row_update_f64(self.c_indptr, self.c_users, self.c_pos, self.ratings, self.est, self.P, self.Q, self._reg,
                                out=self.Q2)
        mark("items")
        ops.nnmf_row_update_f64(self.indptr, self.items, None, self.ratings, self.est, self.Q, self.P, self._reg,
                                out=self.P)
        mark("users")
        self.Q, self.Q2 = self.Q2, self.Q

    def topk(self, k, mask_indptr, mask_indices, users=None):
        """predict() = P[u].Q[i] + bi[i] + bu[u] + mu: the per-user terms do not change the ranking, so the kernel ranks
        P[u].Q[i] + bi[i] and they are added to the returned values in the reference's order."""
        idx, val = ops.score_topk(self.P, self.Q, self.bi, self.F, k, mask_indptr, mask_indices, users=users)
        bu = self.bu if users is None else self.bu[users.long()]
        return idx, (val + bu.unsqueeze(1)) + float(self._mu)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from: P[u].Q[i] + bi[i], without the per-user terms."""
        return ops.score_rank(self.P, self.Q, self.bi, self.F, rel_indptr, rel_items, mask_indptr, mask_indices)

    def get_model_state(self):
        return {"_user_bias": self.bu.cpu().numpy(), "_item_bias": self.bi.cpu().numpy(),
                "_user_embeddings": self.P.cpu().numpy(), "_item_embeddings": self.Q.cpu().numpy()}

    def set_model_state(self, s):
        self.bu, self.bi, self.P, self.Q = (upload(np.asarray(s[key], np.float64), self.device, torch.float64)
                                            for key in ("_user_bias", "_item_bias", "_user_embeddings", "_item_embeddings"))

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))
        self.Q2 = torch.empty_like(self.Q)

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)


class NonNegMF(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    r"""Non-Negative Matrix Factorization (https://ieeexplore.ieee.org/document/6748996) on the H100.

    YAML block as the reference's: NonNegMF: {meta: {...}, epochs, batch_size, factors, lr, reg}; optional keys
    `b200_eval` and `b200_device`.
    """

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "factors", 10, None, None),
            ("_learning_rate", "lr", "lr", 0.001, None, None),
            ("_l_w", "reg", "reg", 0.1, None, None),
        ]
        self.autoset_params()
        if self._batch_size < 1:
            self._batch_size = self._data.transactions
        self._global_mean = np.mean(self._data.sp_i_train_ratings)
        self._device = cuda_device(self._params, "NonNegMF")
        self._model = NonNegMFModel(self._data, len(self._data.users), len(self._data.items), self._global_mean,
                                    self._factors, self._l_w, self._learning_rate, random_seed=self._seed,
                                    device=self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return "NonNegMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        for it in self.iterate(self._epochs):
            self._iteration = it
            self._model.train_step()
            self.evaluate(it)
