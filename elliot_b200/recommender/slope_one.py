"""SlopeOne (Lemire and Maclachlan 2005, "Slope one predictors for online rating-based collaborative filtering") on the
H100.

Mirrors algebric/slope_one/slope_one.py and slope_one_model.py (no parameters, name "SlopeOne", train() = initialize
once and evaluate once):
  freq[i, j] = users with entries for both i and j (explicit 0 ratings included), dev[i, j] = sum_u (r_ui - r_uj) /
  freq[i, j] (0 where freq = 0), user_mean[u] = np.mean of u's ratings, and
  predict(u, c) = user_mean[u] + sum(dev[c, j] for j in Ri) / len(Ri), Ri = u's train items j with freq[c, j] > 0 in
  the order of i_train_dict[u] (user_mean[u] when Ri is empty); train items masked, top k.

On the device (csrc/slope_one.cu): the ratings times 2^s (`knn.exactness_scale`) and the entry pattern are densified to
bf16, so that F = B^T B, M1 = X^T B and M2 = B^T X from the tensor-core GEMM are exact; in row slabs, eb_slope_one_dev_f64
turns them into E = ((M1 - M2) 2^-s) / F in fp64 (NaN where F = 0).  For ratings of that class D = (M1 - M2) 2^-s is the
reference's exact sum, and dev[c, j] = -E[j, c] bit for bit.  eb_slope_one_score_topk_f64 sums -E[j, c] over each user's
train items in dict order with plain fp64 additions (the reference's sum() over np.float64), divides once by the count,
adds the mean and selects the top k; the scores equal the reference's bit for bit.  Other ratings raise ValueError.
`meta.save_weights` writes nothing, as in the reference; `meta.restore` and evaluation-time negative sampling raise
NotImplementedError.
"""
import time

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import TopKRecs, check_free, cuda_device, upload_csr
from .knn import EXACT_LIMIT, SLAB_BYTES, dense_operand, exactness_scale


def dict_order_csr(data):
    """(indptr int64, items int32, ratings float64) of the train ratings, one row per private user, each row in the
    iteration order of `data.i_train_dict[u]` (the order the reference sums in)."""
    n_users = len(data.users)
    if hasattr(data, "_tr"):                                          # the mirror: rows straight from the grouped arrays
        u, i, r = data._tr
        indptr = np.zeros(n_users + 1, np.int64)
        np.cumsum(np.bincount(u, minlength=n_users), out=indptr[1:])
        return indptr, i.astype(np.int32), np.asarray(r, dtype=np.float64)
    rows = [data.i_train_dict.get(u, {}) for u in range(n_users)]
    indptr = np.zeros(n_users + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=indptr[1:])
    items = np.fromiter((j for r in rows for j in r), dtype=np.int32, count=int(indptr[-1]))
    ratings = np.fromiter((v for r in rows for v in r.values()), dtype=np.float64, count=int(indptr[-1]))
    return indptr, items, ratings


class SlopeOneModel:
    """The dict-order train CSR, the deviation matrix E on the device, and the scorer."""

    def __init__(self, data, device="cuda:0"):
        self.device = torch.device(device)
        self.n_users, self.n_items = len(data.users), len(data.items)
        self.indptr, self.items, self.ratings = dict_order_csr(data)
        self.nnz = int(self.indptr[-1])
        self.s = exactness_scale(self.ratings, "SlopeOne needs")
        self.ld = (self.n_items + 7) // 8 * 8
        self.slab_rows = min(max(8, SLAB_BYTES // (12 * max(self.n_items, 1)) // 8 * 8), self.ld)
        self.train = self.E = None

    def working_set(self):
        """(bytes needed at the peak, a description)."""
        g = 2 ** 30
        operands = 2 * self.n_users * self.ld * 2
        E = self.n_items * self.n_items * 8
        slabs = 3 * self.slab_rows * self.n_items * 4
        csr = self.nnz * 8 + (self.n_users + 1) * 8
        return operands + E + slabs + csr, (f"the two bf16 operands {operands / g:.2f} GiB, E {E / g:.2f} GiB, the three "
                                            f"product slabs {slabs / g:.2f} GiB, the train CSR {csr / g:.2f} GiB")

    def initialize(self, mark=None):
        """E.  `mark(phase)`, when given, is called as each phase's work has been queued (upload, operands, products,
        dev), so that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        self.train = self.E = None
        check_free("SlopeOne", self.device, *self.working_set())
        n, U = self.n_items, self.n_users
        self.train = upload_csr(self.indptr, self.items, self.ratings, self.device)
        mark("upload")
        X, s, _ = dense_operand(self.train, U, n, "items", "SlopeOne needs")
        B, _, counts = ops.csr_to_dense_bf16(self.train[0], self.train[1], None, n, col_sq=True)
        if n and float(counts.max().item()) >= EXACT_LIMIT:
            raise ValueError("an item has 2^24 or more entries: the fp32 co-rating counts would not be exact")
        mark("operands")
        self.E = torch.empty((n, n), dtype=torch.float64, device=self.device)
        slab = torch.empty((3, self.slab_rows, n), dtype=torch.float32, device=self.device)
        for j0 in range(0, n, self.slab_rows):
            S = min(self.slab_rows, n - j0)
            F, M1, M2 = slab[0, :S], slab[1, :S], slab[2, :S]
            # rows j0.. of B^T B, X^T B and B^T X: every operand read with users as the K dimension
            ops.gemm_bf16(B[:, j0:], B, S, n, U, a_rows_are_k=True, b_rows_are_k=True, out=F)
            ops.gemm_bf16(X[:, j0:], B, S, n, U, a_rows_are_k=True, b_rows_are_k=True, out=M1)
            ops.gemm_bf16(B[:, j0:], X, S, n, U, a_rows_are_k=True, b_rows_are_k=True, out=M2)
            mark("products")
            ops.slope_one_dev_f64(F, M1, M2, n, s, out=self.E[j0:j0 + S])
            mark("dev")
        del X, B, slab

    def topk(self, k, mask_indptr, mask_indices, users=None):
        return ops.slope_one_score_topk(self.E, self.train, k, mask_indptr, mask_indices, users=users)

    def save_weights(self, path):
        """The reference's SlopeOne never writes weights either."""


class SlopeOne(TopKRecs, RecMixin, BaseRecommenderModel):
    r"""Slope One Predictors for Online Rating-Based Collaborative Filtering (https://arxiv.org/abs/cs/0702144), on the
    H100.  YAML block as the reference's: SlopeOne: {meta: {...}}; optional keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = []
        self.autoset_params()
        if self._restore:
            raise NotImplementedError("meta.restore is not supported for SlopeOne: this build keeps its deviation matrix "
                                      "on the device only")
        self._device = cuda_device(self._params, "SlopeOne")
        self._model = SlopeOneModel(self._data, self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return "SlopeOne"

    def train(self):
        start = time.time()
        self._model.initialize()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The deviation computation has taken: {time.time() - start}")
        self.evaluate()
