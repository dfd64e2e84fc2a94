"""PureSVD (Cremonesi, Koren and Turrin 2010, "Performance of recommender algorithms on top-N recommendation tasks") on
the H100.

Mirrors latent_factor_models/PureSVD/pure_svd.py and pure_svd_model.py (`_params_list`, name, train() = fit once and
evaluate once): sklearn's randomized_svd(sp_i_train, n_components=factors, random_state=seed), user_vec = U and
item_vec = (diag(s) Vt)^T, scores user_vec . item_vec^T with the train items masked, top k.

randomized_svd runs on M = A (the binary train matrix) when num_users >= num_items and on M = A^T otherwise, with
w = factors + 10 columns: the start block Omega = RandomState(seed).normal(size=(columns of M, w)) in float32, n_iter
(7 when factors < 0.1 min(U, I), else 4) power iterations Q <- orth(M Q), Q <- orth(M^T Q), then Q <- orth(M Q),
B = Q^T M and the SVD of B.  This build draws Omega on the host exactly so and runs the rest on the device in fp64
(csrc/pure_svd.cu):
  - M Q and M^T Q are eb_csr_spmm_f64 on the CSRs of A and A^T, uploaded once;
  - orth is pivoted CholeskyQR2: twice, G = X^T X (eb_gram_f64), M = P L^-T (eb_chol_pivoted_f64), X <- X M.  It spans
    the same subspace as sklearn's LU and QR normalisers and keeps the numerical rank (zero columns past it);
  - the SVD of B comes from the eigen-decomposition B B^T = (M^T Q)^T (M^T Q) = W diag(lambda) W^T (eb_sym_eig_f64):
    s = sqrt(lambda), the M-side vectors Q W, and the other side M^T (Q W) = V diag(s), one more product;
  - eb_svd_finish_f64 applies sklearn's svd_flip to the user-side vectors (U when M = A, V when M = A^T) and, when
    M = A^T, forms user_vec = M^T (Q W) diag(1 / s) (0 for singular values at rank-deficiency level) and
    item_vec = (Q W) diag(s).
The first min(factors, min(U, I)) components are kept, as sklearn does.  The tables are fp64 and the scores are
eb_score_topk_f64.  factors + 10 <= 200 (the width eb_gram_f64 takes); more raises ValueError.  `meta.save_weights`,
`meta.restore` and evaluation-time negative sampling raise NotImplementedError.
"""
import time

import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, check_free, cuda_device, upload, upload_csr

OVERSAMPLES = 10                # sklearn's n_oversamples default


def max_factors():
    return ops.svd_max_width() - OVERSAMPLES


def start_block(seed, rows, w):
    """sklearn's _randomized_range_finder start: RandomState(seed).normal(size=(rows, w)) cast to the float32 of A."""
    return np.random.RandomState(seed).normal(size=(rows, w)).astype(np.float32)


class PureSVDModel:
    """Both sides' CSRs on the device, the fit, and the fp64 factor tables."""

    def __init__(self, factors, data, seed, device="cuda:0"):
        self.device = torch.device(device)
        self.factors = int(factors)
        if not 1 <= self.factors <= max_factors():
            raise ValueError(f"factors={factors}: PureSVD supports 1 to {max_factors()} factors here (factors + "
                             f"{OVERSAMPLES} oversamples must fit the {ops.svd_max_width()}-column blocks)")
        A = sp.csr_matrix(data.sp_i_train, dtype=np.float32)
        A.sort_indices()
        self.n_users, self.n_items = A.shape
        self.nnz = A.nnz
        self.w = self.factors + OVERSAMPLES
        self.transpose = self.n_users < self.n_items
        small = min(self.n_users, self.n_items)
        self.n_iter = 7 if self.factors < 0.1 * small else 4
        self.d = min(self.factors, small)
        self.seed = int(seed)
        cols = self.n_users if self.transpose else self.n_items
        self.omega = start_block(self.seed, cols, self.w)
        self._A, self._At = A, A.T.tocsr()
        self._At.sort_indices()
        self.user_vec = self.item_vec = self.s = None

    def working_set(self):
        """(bytes needed at the peak, a description)."""
        g = 2 ** 30
        csr = 2 * (self.nnz * 8 + (self.n_users + self.n_items + 2) * 8)
        blocks = (self.n_users + self.n_items) * self.w * 8 * 2
        tables = (self.n_users + self.n_items) * self.d * 8
        return csr + blocks + tables, (f"both CSRs {csr / g:.2f} GiB, the {self.w}-column blocks {blocks / g:.2f} GiB, "
                                       f"the tables {tables / g:.2f} GiB")

    def _orth(self, X, mark):
        """Pivoted CholeskyQR2 in place."""
        for _ in range(2):
            G = ops.gram_f64(X, self.w)
            ops.tall_times_small_f64(X, ops.chol_pivoted_f64(G), out=X)
        mark("orth")
        return X

    def train_step(self, mark=None):
        """The fit.  `mark(phase)`, when given, is called as each phase's work has been queued (upload, spmm, orth,
        eig, finish), so that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        self.user_vec = self.item_vec = self.s = None
        check_free("PureSVD", self.device, *self.working_set())
        dev = self.device
        a = upload_csr(self._A.indptr, self._A.indices, self._A.data, dev)
        at = upload_csr(self._At.indptr, self._At.indices, self._At.data, dev)
        Mc, MTc = (at, a) if self.transpose else (a, at)
        Q = upload(self.omega, dev, torch.float64)
        Y = torch.empty((Mc[0].numel() - 1, self.w), dtype=torch.float64, device=dev)
        mark("upload")

        def spmm(csr, X, out=None):
            out = ops.csr_spmm_f64(csr, X, out=out)
            mark("spmm")
            return out
        for _ in range(self.n_iter):
            self._orth(spmm(Mc, Q, out=Y), mark)
            self._orth(spmm(MTc, Y, out=Q), mark)
        self._orth(spmm(Mc, Q, out=Y), mark)
        Z = spmm(MTc, Y, out=Q)                                   # B^T = M^T Q
        evals, W = ops.sym_eig_f64(ops.gram_f64(Z, self.w))
        UM = ops.tall_times_small_f64(Y, W[:, :self.d].contiguous())
        mark("eig")
        other = spmm(MTc, UM)
        user, item = (other, UM) if self.transpose else (UM, other)
        self.s = ops.svd_finish_f64(evals, user, item, self.transpose)
        mark("finish")
        self.user_vec, self.item_vec = user, item

    def topk(self, k, mask_indptr, mask_indices, users=None):
        return ops.score_topk(self.user_vec, self.item_vec, None, self.d, k, mask_indptr, mask_indices, users=users)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        return ops.score_rank(self.user_vec, self.item_vec, None, self.d, rel_indptr, rel_items, mask_indptr, mask_indices)


class PureSVD(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    r"""PureSVD (https://link.springer.com/chapter/10.1007/978-0-387-85820-3_5), on the H100.  YAML block as the
    reference's: PureSVD: {meta: {...}, factors, seed}; optional keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "factors", 10, None, None)
        ]
        self.autoset_params()
        if self._save_weights or self._restore:
            raise NotImplementedError("meta.save_weights / meta.restore are not supported for PureSVD: this build keeps "
                                      "its fp64 factor tables on the device only")
        self._device = cuda_device(self._params, "PureSVD")
        self._model = PureSVDModel(self._factors, self._data, self._seed, self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return f"PureSVD_{self.get_params_shortcut()}"

    def train(self):
        start = time.time()
        self._model.train_step()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The PureSVD fit has taken: {time.time() - start}")
        self.evaluate()
