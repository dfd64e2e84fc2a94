"""EASE^R (Steck 2019, "Embarrassingly shallow autoencoders for sparse data") on the H100.

Mirrors autoencoders/EASE_R/ease_r.py (`_params_list`, name, logging, train() = build once and evaluate once):
  X     = sp_i_train_ratings (float32 ratings, not ones);
  G     = X^T X with the diagonal replaced by fp32(count_j + l2_norm), count_j the number of train ratings of item j;
  P     = G^-1;
  B     = P / -diag(P) column by column, B_jj = 0, in float32;
  preds = X . B, train items masked, top k.
`neighborhood` is parsed and, as in the reference, not used.

On the device: the Gram matrix comes exact from the tensor-core GEMM of kNN (`dense_operand` / `gram_slabs`, the same
`exactness_scale` refusal), slab by slab into an fp64 matrix (eb_ease_normal_f64), which is inverted in place in fp64
(eb_inverse_f64: blocked Gauss-Jordan with partial pivoting, because with explicit ratings G is usually indefinite).
B is written in fp32 (eb_ease_weights_f32), the reference's dtype, and the fp64 matrix is freed.  Scoring is the fused
masked top-k of kNN with a dense B (eb_dense_score_topk_f32): int64 fixed-point sums, so the scores do not depend on the
order of the terms; the dense `_preds` matrix of the reference is never formed.  `meta.save_weights`, `meta.restore` and
evaluation-time negative sampling raise NotImplementedError.  The DataSet is not modified.
"""
import time

import numpy as np
import torch

from .. import ops
from .._lib import EbError
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import TopKRecs, check_free, cuda_device, upload, upload_csr
from .knn import SLAB_BYTES, _bound, dense_operand, frac_bits, gram_slabs


class EASEModel:
    """The item-item weight matrix B (fp32 [n_items][n_items] on the device) and its scoring."""

    def __init__(self, data, l2_norm, device):
        self.l2_norm = l2_norm
        self.device = torch.device(device)
        m = data.sp_i_train_ratings.tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        self.urm = upload_csr(m.indptr, m.indices, m.data, self.device)
        self.n_users, self.n_items = m.shape
        # ease_r.py:86: np.ediff1d(X.tocsc().indptr), the number of stored ratings per item
        self.count = upload(np.bincount(m.indices, minlength=self.n_items), self.device, torch.int32)
        self.B = None

    def working_set(self):
        """(bytes needed at the peak, a description): the fp64 matrix plus the larger of (dense bf16 ratings + one Gram
        slab) and the fp32 B."""
        n, U = self.n_items, self.n_users
        a = 8 * n * n
        x = 2 * U * ((n + 7) // 8 * 8) + min(SLAB_BYTES, 4 * n * ((n + 7) // 8 * 8))
        b = 4 * n * n
        g = 2 ** 30
        return a + max(x, b), (f"the fp64 normal matrix {a / g:.1f} GiB ({n} x {n} x 8 bytes), then either the dense bf16 "
                               f"ratings and a Gram slab {x / g:.1f} GiB or the fp32 weights {b / g:.1f} GiB")

    def initialize(self, mark=None):
        """B.  `mark(phase)`, when given, is called as each phase's work has been queued (gram, inverse, weights), so
        that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        n = self.n_items
        self.B = None
        check_free("EASER", self.device, *self.working_set())
        X, s, _ = dense_operand(self.urm, self.n_users, n, "items", who="EASER needs")
        A = torch.empty((n, n), dtype=torch.float64, device=self.device)
        for j0, C in gram_slabs(X, self.n_users, n, "items"):
            ops.ease_normal_f64(C, j0, self.count, self.l2_norm, 4.0 ** -s, A)
        del X, C
        mark("gram")
        try:
            ops.inverse_f64(A)
            mark("inverse")
            self.B = ops.ease_weights_f32(A)
        except EbError as e:
            if "error -4" not in str(e):
                raise
            raise ValueError(f"EASER: the normal matrix X^T X with diagonal item_popularity + l2_norm (l2_norm="
                             f"{self.l2_norm}) is singular to working precision; a larger l2_norm makes it regular ({e})") \
                from None
        del A
        self.frac_bits = frac_bits(_bound(self.urm, (None, None, self.B.view(-1))))
        mark("weights")

    def topk(self, k, mask_indptr, mask_indices, users=None, user_begin=0, n_sel=None):
        return ops.dense_score_topk(self.urm, self.B, k, self.frac_bits, mask_indptr, mask_indices, users=users,
                                    user_begin=user_begin, n_sel=n_sel)


class EASER(TopKRecs, RecMixin, BaseRecommenderModel):
    r"""Embarrassingly shallow autoencoders for sparse data (https://dl.acm.org/doi/abs/10.1145/3308558.3313710), on the
    H100.  YAML block as the reference's: EASER: {meta: {...}, neighborhood, l2_norm}; optional keys `b200_eval` and
    `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_neighborhood", "neighborhood", "neighborhood", -1, int, None),
            ("_l2_norm", "l2_norm", "l2_norm", 1e3, float, None)
        ]
        self.autoset_params()
        if self._neighborhood == -1:
            self._neighborhood = self._data.num_items
        if self._save_weights or self._restore:
            raise NotImplementedError("meta.save_weights / meta.restore are not supported for EASER: the reference "
                                      "pickles the dense prediction matrix, which this build never forms")
        self._device = cuda_device(self._params, "EASER")
        self._model = EASEModel(self._data, self._l2_norm, self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return f"EASER_{self.get_params_shortcut()}"

    def train(self):
        start = time.time()
        self._model.initialize()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The similarity computation has taken: {time.time() - start}")
        self.evaluate()
