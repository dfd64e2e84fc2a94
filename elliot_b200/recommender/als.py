"""iALS and WRMF (implicit alternating least squares) on the H100.

Mirrors latent_factor_models/iALS/iALS.py + iALS_model.py and latent_factor_models/WRMF/wrmf.py + wrmf_model.py
(`_params_list`, name, train() = one alternating step and one evaluation per epoch).  Both models solve, for every user
and then every item, the normal equations
    x_r = (G + sum_{e in row r} w_e y_e y_e^T + reg I)^-1 sum_{e in row r} c_e y_e,   G = Y^T Y (users) or X^T X (items),
and differ in the weights and in which G the item half sees:
  iALS:  C = 1 + alpha r (linear) or 1 + alpha log(1 + r / epsilon) (log), float32 as the reference computes it;
         w = C - 1, c = C; X^T X is taken from the NEW X; items without train entries keep their initial rows.
  WRMF:  C = alpha r (float32), w = C, c = C + 1 where C != 0; X^T X is taken BEFORE the user half (stale, as
         wrmf_model.py:42); every item is solved, so an item without entries gets 0.
The factors start as the reference's: X then Y drawn from normal(scale=0.01) on the global numpy stream that the model
seed initialised.  The confidences are computed on the host once, with the reference's numpy expressions and dtypes, from
a COPY of `sp_i_train`: the reference's iALS rewrites the DataSet's `sp_i_train` in place (iALS_model.py:25-29), which
this build does not do.

On the device: fp64 tables, eb_gram_f64 for G and eb_als_solve_f64 for each half (rank-k updates on the fp64 tensor
cores, Cholesky in shared memory); rows are visited longest first (`order`, built once per side), which balances the load
and does not change the result.  Scoring is eb_score_topk_f64 with no bias.  `meta.save_weights`, `meta.restore` and
evaluation-time negative sampling raise NotImplementedError.
"""
import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from .._lib import EbError
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, cuda_device, upload

MAX_FACTORS = 200              # the top of the reference's own search range (config_files/recsys_config.yml, iALS block)


def ials_confidences(values, alpha, epsilon, scaling):
    """(w, c) of iALS_model.py:25-29 and :47-51 for the float32 train values, computed in float32 as the reference does
    (C = 1 + alpha * r, or 1 + alpha * log(1 + r / epsilon); w = C - 1; c = C), returned as fp64."""
    C = np.array(values, dtype=np.float32)
    if scaling == "linear":
        C = 1.0 + alpha * C
    elif scaling == "log":
        C = 1.0 + alpha * np.log(1.0 + C / epsilon)
    return (C - 1).astype(np.float64), C.astype(np.float64)


def wrmf_confidences(m, alpha):
    """(w, c) of wrmf_model.py:25 and :45-49 for the float32 train CSR m: C = alpha * m (float32), w = C, and
    c = C + 1 (the fp64 identity added to the float32 C) on the entries where C != 0, else 0."""
    C = (alpha * m).data
    w = C.astype(np.float64)
    return w, np.where(C != 0, w + 1.0, 0.0)


class ALSModel:
    """The factor model both classes share: fp64 tables and both sides' CSRs on the device."""

    def __init__(self, kind, factors, data, alpha, reg, epsilon=1.0, scaling="linear", device="cuda:0"):
        self.kind, self.d, self.alpha, self.reg = kind, int(factors), alpha, float(reg)
        self.device = torch.device(device)
        nu, ni = len(data.users), len(data.items)
        # iALS_model.py:34-35, wrmf_model.py:30-33: X then Y, from the stream init_charger seeded
        X0 = np.random.normal(scale=0.01, size=(nu, self.d))
        Y0 = np.random.normal(scale=0.01, size=(ni, self.d))
        m = data.sp_i_train.tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        if kind == "iALS":
            w, c = ials_confidences(m.data, alpha, epsilon, scaling)
        else:
            w, c = wrmf_confidences(m, alpha)
        self.w_host, self.c_host = w, c
        dev = self.device
        # item side: the transpose, its entries permuted along (users ascending within an item)
        nnz = m.nnz
        t = sp.csr_matrix((np.arange(nnz, dtype=np.int64), m.indices, m.indptr), shape=m.shape).tocsc()
        perm = t.data
        lens_u, lens_i = np.diff(m.indptr), np.diff(t.indptr)
        order_u = np.argsort(-lens_u, kind="stable")
        order_i = np.argsort(-lens_i, kind="stable")
        if kind == "iALS":
            order_i = order_i[lens_i[order_i] > 0]          # iALS_model.py:37-38: only warm items are solved
        self.users = (upload(m.indptr, dev, torch.int64), upload(m.indices, dev, torch.int32), upload(w, dev, torch.float64),
                      upload(c, dev, torch.float64), upload(order_u, dev, torch.int32))
        self.items = (upload(t.indptr, dev, torch.int64), upload(t.indices, dev, torch.int32), upload(w[perm], dev, torch.float64),
                      upload(c[perm], dev, torch.float64), upload(order_i, dev, torch.int32))
        self.X, self.Y = upload(X0, dev, torch.float64), upload(Y0, dev, torch.float64)
        self.G = torch.empty((self.d, self.d), dtype=torch.float64, device=self.device)
        self.G2 = torch.empty_like(self.G)

    def _solve(self, G, other, side, out):
        indptr, indices, w, c, order = side
        try:
            ops.als_solve_f64(G, other, self.d, indptr, indices, w, c, order, self.reg, out)
        except EbError as e:
            if "error -4" not in str(e):
                raise
            raise ValueError(f"{self.kind}: a normal matrix is not positive definite (alpha={self.alpha}, reg={self.reg}); "
                             f"this build needs reg > 0 and confidences that keep every weight w = C - 1 (iALS) or "
                             f"C (WRMF) >= 0, for example alpha >= 0 ({e})") from None

    def train_step(self, mark=None):
        """One alternating step: iALS_model.py:40-65 / wrmf_model.py:40-58.  `mark(phase)`, when given, is called as
        each phase's work has been queued (iALS: gram, user_half, gram, item_half; WRMF: gram, gram, user_half,
        item_half), so that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        if self.kind == "iALS":
            ops.gram_f64(self.Y, self.d, out=self.G)
            mark("gram")
            self._solve(self.G, self.Y, self.users, self.X)
            mark("user_half")
            ops.gram_f64(self.X, self.d, out=self.G)
            mark("gram")
            self._solve(self.G, self.X, self.items, self.Y)
            mark("item_half")
        else:
            ops.gram_f64(self.Y, self.d, out=self.G)
            mark("gram")
            ops.gram_f64(self.X, self.d, out=self.G2)         # wrmf_model.py:42: X^T X before the user half
            mark("gram")
            self._solve(self.G, self.Y, self.users, self.X)
            mark("user_half")
            self._solve(self.G2, self.X, self.items, self.Y)
            mark("item_half")

    def topk(self, k, mask_indptr, mask_indices, users=None):
        return ops.score_topk(self.X, self.Y, None, self.d, k, mask_indptr, mask_indices, users=users)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        return ops.score_rank(self.X, self.Y, None, self.d, rel_indptr, rel_items, mask_indptr, mask_indices)


class _ALS(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    _kind = None

    def _check(self):
        if not 1 <= int(self._factors) <= MAX_FACTORS:
            raise ValueError(f"factors={self._factors}: {self._kind} supports 1 to {MAX_FACTORS} factors "
                             f"({MAX_FACTORS} is the top of the reference's own search range)")
        if self._save_weights or self._restore:
            raise NotImplementedError(f"meta.save_weights / meta.restore are not supported for {self._kind}: the "
                                      f"reference pickles the dense prediction matrix, which this build never forms")
        self._device = cuda_device(self._params, type(self).__name__)

    @property
    def name(self):
        return f"{self._kind}_{self.get_base_params_shortcut()}_{self.get_params_shortcut()}"

    def train(self):
        for it in self.iterate(self._epochs):
            self._model.train_step()
            self.evaluate(it)


class iALS(_ALS):
    r"""Collaborative filtering for implicit feedback datasets (https://ieeexplore.ieee.org/document/4781121), on the
    H100.  YAML block as the reference's: iALS: {meta: {...}, epochs, factors, alpha, epsilon, reg, scaling};
    optional keys `b200_eval` and `b200_device`."""
    _kind = "iALS"

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "factors", 10, int, None),
            ("_alpha", "alpha", "alpha", 1, float, None),
            ("_epsilon", "epsilon", "epsilon", 1, float, None),
            ("_reg", "reg", "reg", 0.1, float, None),
            ("_scaling", "scaling", "scaling", "linear", None, None)
        ]
        self.autoset_params()
        self._check()
        self._model = ALSModel("iALS", self._factors, self._data, self._alpha, self._reg, self._epsilon, self._scaling,
                               self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)


class WRMF(_ALS):
    r"""Weighted regularised matrix factorisation (https://ieeexplore.ieee.org/document/4781121), on the H100.  YAML
    block as the reference's: WRMF: {meta: {...}, epochs, factors, alpha, reg}; optional keys `b200_eval` and
    `b200_device`."""
    _kind = "WRMF"

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "factors", 10, None, None),
            ("_alpha", "alpha", "alpha", 1, None, None),
            ("_reg", "reg", "reg", 0.1, None, None)
        ]
        self.autoset_params()
        self._check()
        self._model = ALSModel("WRMF", self._factors, self._data, self._alpha, self._reg, device=self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
