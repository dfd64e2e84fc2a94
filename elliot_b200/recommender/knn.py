"""ItemKNN / UserKNN, standard implementation, on the H100.

Mirrors knn/item_knn/item_knn.py:45-125 and knn/user_knn/user_knn.py (`_params_list`, name, logging, train() = build once
and evaluate once) and the two `Similarity` classes (item_knn_similarity.py, user_knn_similarity.py):
  URM     = sp_i_train_ratings (sp_i_train with `implicit: True`);
  S       = cosine_similarity(URM.T) or URM.T @ URM (items), resp. the same over users;
  W       = per column the `neighbors` largest nonzero similarities (the row itself included), CSC fp32;
  preds   = URM . W (items) or W . URM (users); train items masked, top k.

On the device: the ratings are densified to bf16 times 2^s (`exactness_scale`), so the Gram matrix from the tensor-core
GEMM is exact; it is computed in row slabs, and each slab goes straight into the neighbour kernel.  The neighbour lists,
transposed into W's CSR by an index sort, feed the fused sparse-product + masked top-k kernel; the dense `_preds` matrix of
the reference is never formed.  Other similarities, `implementation: aiolli`, `meta.save_weights` and `meta.restore`
are not supported and raise NotImplementedError.
"""
import math
import time

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import TopKRecs, cuda_device, upload_csr

SIMILARITIES = ("cosine", "dot")
SLAB_BYTES = 2 << 30            # fp32 Gram rows computed per GEMM call
EXACT_LIMIT = float(1 << 24)    # every integer below it is exact in fp32


def exactness_scale(values, who="ItemKNN/UserKNN need"):
    """Smallest s in 0..4 such that every value * 2^s is an integer of magnitude <= 256.  Refuses other data: the bf16
    Gram is exact only for such values, and there is no other path."""
    v = np.asarray(values, dtype=np.float64)
    for s in range(5):
        x = v * (1 << s)
        if np.all(x == np.round(x)) and np.abs(x).max(initial=0.0) <= 256:
            return s
    raise ValueError(f"{who} ratings that become integers of magnitude <= 256 when multiplied by 1, 2, 4, 8 "
                     "or 16 (for example 1-5, half stars, implicit ones); these ratings do not, and the tensor-core "
                     "Gram matrix would not be exact")


def frac_bits(bound):
    """Fixed-point fraction bits for sums of terms whose absolute values add up to at most `bound`: bound * 2^f < 2^61."""
    if not bound > 0:
        return 0
    return max(-1000, min(1000, 61 - math.frexp(float(bound))[1]))


def _row_abs_sums(indptr, values):
    cs = torch.cat([torch.zeros(1, dtype=torch.float64, device=values.device), torch.cumsum(values.double().abs(), 0)])
    return cs[indptr[1:]] - cs[indptr[:-1]]


def _bound(A, B):
    """max_p sum_q |A[p, q]| * max |B|"""
    if A[2].numel() == 0 or B[2].numel() == 0:
        return 0.0
    return float(_row_abs_sums(A[0], A[2]).max().item()) * float(B[2].abs().max().item())


def dense_operand(urm, n_users, n_items, over, who="ItemKNN/UserKNN need"):
    """The exact bf16 Gram operand of the ratings: (X = ratings * 2^s as bf16 [n_users][pad8(n_items)], s, the Gram
    diagonal as fp32).  urm: (indptr, indices, values) on the device.  Refuses ratings for which the tensor-core Gram
    would not be exact."""
    indptr, indices, values = urm
    s = exactness_scale(values.cpu().numpy(), who)
    dev = indptr.device
    ld = (n_items + 7) // 8 * 8
    need = n_users * ld * 2
    free = torch.cuda.mem_get_info(dev)[0]
    if need > free:
        raise MemoryError(f"the dense bf16 rating matrix needs {need / 2**30:.1f} GiB ({n_users} x {ld} x 2 bytes) and "
                          f"{free / 2**30:.1f} GiB are free on {dev}; a sparse Gram for catalogues of this size is not built")
    items = over == "items"
    X, rs, cs = ops.csr_to_dense_bf16(indptr, indices, values, n_items, scale=float(1 << s), row_sq=not items, col_sq=items)
    diag = cs if items else rs
    n = n_items if items else n_users
    if n and float(diag.max().item()) >= EXACT_LIMIT:
        raise ValueError(f"a squared {'item' if items else 'user'} norm of the scaled ratings reaches 2^24: the fp32 Gram "
                         f"matrix would not be exact")
    return X, s, diag


def gram_slabs(X, n_users, n_items, over, slab_rows=None):
    """The exact fp32 Gram matrix of dense_operand()'s X (X^T X for over="items", X X^T for "users"), in row slabs: yields
    (j0, C) with C the rows j0 .. j0 + C.shape[0], in order.  C is one buffer, overwritten by the next slab."""
    items = over == "items"
    n = n_items if items else n_users
    if slab_rows is None:
        slab_rows = max(8, SLAB_BYTES // (4 * max(n, 1)) // 8 * 8)
    slab_rows = min(slab_rows, (n + 7) // 8 * 8)
    assert slab_rows % 8 == 0, "slab starts must stay 16-byte aligned"
    slab = torch.empty((slab_rows, n), dtype=torch.float32, device=X.device)
    for j0 in range(0, n, slab_rows):
        S = min(slab_rows, n - j0)
        C = slab[:S]
        if items:       # rows j0.. of X^T X: both operands are X itself, read with users as the K dimension
            ops.gemm_bf16(X[:, j0:], X, S, n, n_users, a_rows_are_k=True, b_rows_are_k=True, out=C)
        else:           # rows j0.. of X X^T
            ops.gemm_bf16(X[j0:], X, S, n, n_items, out=C)
        yield j0, C


def neighbours(urm, n_users, n_items, over, k, cosine, slab_rows=None, mark=None):
    """Neighbour lists of every item (over="items") or user (over="users").  urm: (indptr, indices, values) on the device.
    Returns (idx int32 [n][k], val fp32 [n][k]): value desc then index asc, -1 / 0 padded.  `mark(phase)`, when given, is
    called as each phase's work has been queued (densify, then gram and neighbours per slab)."""
    mark = mark or (lambda phase: None)
    X, s, diag = dense_operand(urm, n_users, n_items, over)
    mark("densify")
    n = n_items if over == "items" else n_users
    idx = torch.empty((n, k), dtype=torch.int32, device=X.device)
    val = torch.empty((n, k), dtype=torch.float32, device=X.device)
    for j0, C in gram_slabs(X, n_users, n_items, over, slab_rows):
        mark("gram")
        i, v, _ = ops.knn_neighbors(C, n, j0, diag, k, cosine=cosine, dot_scale=4.0 ** -s)
        idx[j0:j0 + C.shape[0]], val[j0:j0 + C.shape[0]] = i, v
        mark("neighbours")
    return idx, val


def transpose_lists(idx, val):
    """W in CSR form from neighbour lists: row x lists every y that has x among its neighbours, sorted by y, with the
    value x has in y's list (the reference's CSC W, item_knn_similarity.py:76-77, read by rows)."""
    n = idx.shape[0]
    ok = idx >= 0
    x = idx[ok].long()
    y = torch.arange(n, device=idx.device).unsqueeze(1).expand_as(idx)[ok]
    order = torch.argsort(x * n + y)
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=idx.device)
    indptr[1:] = torch.cumsum(torch.bincount(x, minlength=n), 0)
    return indptr, y[order].to(torch.int32).contiguous(), val[ok][order].contiguous()


class KNNModel:
    """The similarity model both classes share (the reference's `Similarity`, standard implementation)."""

    def __init__(self, data, num_neighbors, similarity, implicit, over, device):
        self._data, self._k, self._similarity, self._implicit, self._over = data, num_neighbors, similarity, implicit, over
        self.device = torch.device(device)
        m = (data.sp_i_train if implicit else data.sp_i_train_ratings).tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        self.urm = upload_csr(m.indptr, m.indices, m.data, self.device)
        self.n_users, self.n_items = m.shape
        self.A = self.B = None

    def initialize(self, mark=None):
        """W.  `mark(phase)`, when given, is called as each phase's work has been queued (densify, gram, neighbours,
        transpose), so that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        if not 1 <= self._k <= 1024:
            raise ValueError(f"neighbors={self._k}: 1 to 1024 are supported")
        self.A = self.B = None
        n = self.n_items if self._over == "items" else self.n_users
        idx, val = neighbours(self.urm, self.n_users, self.n_items, self._over, min(self._k, max(n, 1)),
                              self._similarity == "cosine", mark=mark)
        W = transpose_lists(idx, val)
        self.A, self.B = (self.urm, W) if self._over == "items" else (W, self.urm)
        self.frac_bits = frac_bits(_bound(self.A, self.B))
        mark("transpose")

    def topk(self, k, mask_indptr, mask_indices, users=None, user_begin=0, n_sel=None):
        return ops.knn_score_topk(self.A, self.B, self.n_items, k, self.frac_bits, mask_indptr, mask_indices, users=users,
                                  user_begin=user_begin, n_sel=n_sel)


class _KNN(TopKRecs, RecMixin, BaseRecommenderModel):
    _over = None

    def _setup(self):
        self._params_list = [
            ("_num_neighbors", "neighbors", "nn", 40, int, None),
            ("_similarity", "similarity", "sim", "cosine", None, None),
            ("_implementation", "implementation", "imp", "standard", None, None),
            ("_implicit", "implicit", "bin", False, None, None),
            ("_shrink", "shrink", "shrink", 0, None, None),
            ("_normalize", "normalize", "norm", True, None, None),
            ("_asymmetric_alpha", "asymmetric_alpha", "asymalpha", False, None, lambda x: x if x else ""),
            ("_tversky_alpha", "tversky_alpha", "tvalpha", False, None, lambda x: x if x else ""),
            ("_tversky_beta", "tversky_beta", "tvbeta", False, None, lambda x: x if x else ""),
            ("_row_weights", "row_weights", "rweights", None, None, lambda x: x if x else "")
        ]
        self.autoset_params()
        if self._implementation == "aiolli":
            raise NotImplementedError("implementation: aiolli is not supported by elliot_b200 (standard only)")
        if self._similarity not in SIMILARITIES:
            raise NotImplementedError(f"similarity: {self._similarity} is not supported by elliot_b200 "
                                      f"(supported: {', '.join(SIMILARITIES)})")
        if self._save_weights or self._restore:
            raise NotImplementedError("meta.save_weights / meta.restore are not supported for ItemKNN/UserKNN: the "
                                      "reference pickles the dense prediction matrix, which this build never forms")
        if (not self._normalize) or self._asymmetric_alpha or self._tversky_alpha or self._tversky_beta or \
                self._row_weights or self._shrink:
            self.logger.info("Options normalize, asymmetric_alpha, tversky_alpha, tversky_beta, row_weights are ignored "
                             "with standard implementation. Try with implementation: aiolli")
        self._device = cuda_device(self._params, type(self).__name__)
        self._model = KNNModel(self._data, self._num_neighbors, self._similarity, self._implicit, self._over, self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return f"{type(self).__name__}_{self.get_params_shortcut()}"

    def train(self):
        start = time.time()
        self._model.initialize()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The similarity computation has taken: {time.time() - start}")
        self.logger.info(f"Transactions: {self._data.transactions}")
        self.evaluate()


class ItemKNN(_KNN):
    r"""Amazon.com recommendations: item-to-item collaborative filtering (http://ieeexplore.ieee.org/document/1167344/),
    on the H100.  YAML block as the reference's: ItemKNN: {meta: {...}, neighbors, similarity, implicit, ...};
    optional keys `b200_eval` and `b200_device`."""
    _over = "items"

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._setup()


class UserKNN(_KNN):
    r"""GroupLens: an open architecture for collaborative filtering of netnews (https://dl.acm.org/doi/10.1145/192844.192905),
    on the H100.  YAML block as the reference's: UserKNN: {meta: {...}, neighbors, similarity, implicit, ...};
    optional keys `b200_eval` and `b200_device`."""
    _over = "users"

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._setup()
