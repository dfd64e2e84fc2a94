"""SLIM (Ning and Karypis 2011, "SLIM: Sparse linear methods for top-n recommender systems"; Levy and Jack 2013) on
the H100.

Mirrors latent_factor_models/Slim/slim.py and slim_model.py (`_params_list`, name, train() = fit once and evaluate
once): per item p one sklearn ElasticNet(alpha, l1_ratio, positive=True, fit_intercept=False, selection='random',
max_iter=100, tol=1e-4, random_state=seed) of y = X[:, p] on X = sp_i_train_ratings (float32) with user row p zeroed
(the reference zeroes the CSR row it indexes with the item id; item column p stays, so item p regresses on itself too);
then per column p of W the min(nnz - 1, neighborhood) largest coefficients; preds = X . W (float32), train items
masked, top k.

Every elastic net runs on the device at once (csrc/slim.cu: one warp per item, the reference's float32 coordinate
updates and xorshift order), W is built on the device, and the scores are ops.rp3_score_topk, SciPy's float32 csr * csr
order.  The selections break exact ties by the lower index, which the reference leaves to np.argpartition.  A column
without nonzero coefficients stays empty, as in the reference.  The reference needs num_items <= num_users (it fails
with an IndexError otherwise); this build raises ValueError.  `meta.save_weights`, `meta.restore` and evaluation-time
negative sampling raise NotImplementedError (the reference's get_model_state reads an `_A_tilde` it never sets)."""
import time

import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import TopKRecs, check_free, cuda_device, upload_csr
from .rp3beta import sparse_score_topk


def seed_state(seed):
    """The xorshift state every ElasticNet fit starts from: sparse_enet_coordinate_descent draws
    rng.randint(0, 2**31 - 1) from check_random_state(seed), a fresh RandomState(seed) per fit."""
    return int(np.random.RandomState(seed).randint(0, 2 ** 31 - 1))


class SlimModel:
    """W (a CSR on the device), the per-item solver results, and the scoring."""

    def __init__(self, data, l1_ratio, alpha, neighborhood, seed, device):
        self.device = torch.device(device)
        self.R = sp.csr_matrix(data.sp_i_train_ratings, dtype=np.float32)
        self.n_users, self.n_items = self.R.shape
        if self.n_items > self.n_users:
            raise ValueError(f"SLIM zeroes user row p while fitting item p, so it needs num_items <= num_users; got "
                             f"{self.n_items} items and {self.n_users} users")
        self.k = int(neighborhood)
        if self.k < 1:
            raise ValueError(f"neighborhood={neighborhood}: a positive number of neighbours")
        self.alpha, self.l1_ratio, self.seed = float(alpha), float(l1_ratio), int(seed)
        if not self.alpha * self.l1_ratio > 0:
            raise ValueError(f"alpha={alpha}, l1_ratio={l1_ratio}: SLIM needs a positive L1 penalty")
        # the ElasticNet's penalties, formed in double and passed to the float32 solver
        self.l1 = float(np.float32(self.alpha * self.l1_ratio * self.n_users))
        self.l2 = float(np.float32(self.alpha * (1.0 - self.l1_ratio) * self.n_users))
        self.urm = upload_csr(self.R.indptr, self.R.indices, self.R.data, self.device)
        self.W = None
        self.coef_t = self.n_iter = self.gap = self.nnz = None

    def working_set(self, slots, shared):
        """(bytes needed at the peak, a description)."""
        n, U, nnz = self.n_items, self.n_users, self.R.nnz
        g = 2 ** 30
        coef = n * n * 4
        solver = ops.slim_workspace_bytes(U, n, slots, shared)
        weights = n * n * 8 + n * n + nnz * 8 + n * 64    # the dropped copy, the list columns, keep flags, keys
        operands = 2 * (nnz * 8 + (max(n, U) + 1) * 8)
        return coef + solver + weights + operands, (f"the coefficients {coef / g:.1f} GiB ({n} x {n}), the solver rows "
                                                    f"{solver / g:.1f} GiB ({slots} problems at once), W's assembly "
                                                    f"{weights / g:.1f} GiB")

    def initialize(self, shared_residual=None, slots=None, mark=None):
        """W.  `mark(phase)`, when given, is called as each phase's work has been queued (operands, fit, weights), so
        that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        self.W = self.coef_t = self.n_iter = self.gap = self.nnz = None
        shared = ops.slim_shared_residual_fits(self.n_users) if shared_residual is None else bool(shared_residual)
        cap = ops.slim_slots(self.n_users, shared)
        slots = cap if slots is None else max(1, min(int(slots), cap))
        check_free("SLIM", self.device, *self.working_set(slots, shared))
        C = self.R.tocsc()
        C.sort_indices()
        csc = upload_csr(C.indptr, C.indices, C.data, self.device)
        csr = (self.urm[0], self.urm[1])
        mark("operands")
        self.coef_t, self.n_iter, self.gap, self.nnz, drop = ops.slim_fit(
            csc, csr, self.n_users, self.n_items, self.l1, self.l2, seed_state(self.seed), self.k,
            shared_residual=shared, slots=slots)
        mark("fit")
        self.W = ops.slim_weights(self.coef_t, drop, self.nnz, self.k)
        mark("weights")

    def topk(self, k, mask_indptr, mask_indices, users=None, user_begin=0, n_sel=None):
        return sparse_score_topk(self.urm, self.W, self.n_items, k, mask_indptr, mask_indices, users, user_begin, n_sel)


class Slim(TopKRecs, RecMixin, BaseRecommenderModel):
    r"""Sparse Linear Methods (SLIM) item model, one elastic net per item
    (http://glaros.dtc.umn.edu/gkhome/fetch/papers/SLIM2011icdm.pdf), on the H100.  YAML block as the reference's:
    Slim: {meta: {...}, l1_ratio, alpha, neighborhood}; optional keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_l1_ratio", "l1_ratio", "l1", 0.001, float, None),
            ("_alpha", "alpha", "alpha", 0.001, float, None),
            ("_neighborhood", "neighborhood", "neighborhood", 10, int, None)
        ]
        self.autoset_params()
        if self._save_weights or self._restore:
            raise NotImplementedError("meta.save_weights / meta.restore are not supported for Slim: the reference's "
                                      "model state reads an `_A_tilde` it never sets")
        self._device = cuda_device(self._params, "Slim")
        self._model = SlimModel(self._data, self._l1_ratio, self._alpha, self._neighborhood, self._seed, self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return f"Slim_{self.get_base_params_shortcut()}_{self.get_params_shortcut()}"

    def train(self):
        start = time.time()
        self._model.initialize()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The SLIM fit has taken: {time.time() - start}")
        self.evaluate()
