"""RP3beta (Paudel et al. 2017, "Updatable, accurate, diverse, and scalable recommendations for interactive
applications") on the H100.

Mirrors graph_based/RP3beta/rp3beta.py (`_params_list`, name, train() = build once and evaluate once):
  R       = sp_i_train_ratings (float32, stored order);
  Pui     = R with rows l1-normalised;  Piu = R^T binarised with rows l1-normalised;
  degree  = fp32 popularity ** -beta (0 for items without ratings);  alpha != 1 raises Pui and Piu to alpha;
  S_i     = Piu[i] . Pui (float32) times degree in fp64, diagonal zeroed, its `neighborhood` largest nonzero values;
  W       = S, rows l1-normalised if normalize_similarity, then per column its `neighborhood` largest nonzero values;
  preds   = R . W (float32), train items masked, top k.

The O(nnz) elementwise steps (Pui, Piu, degree, the powers) run on the host with the reference's numpy expressions and
dtypes.  The sparse products are new CUDA (csrc/rp3.cu) that sums every output column in SciPy's order with one
rounded product and one rounded add per term, so the similarity values and the scores equal the reference's bit for bit;
the selections break exact ties by the lower index, which the reference leaves to np.argsort.  The dense `_preds`
matrix of the reference is never formed.  `meta.save_weights`, `meta.restore` and evaluation-time negative sampling
raise NotImplementedError.  The DataSet is not modified.
"""
import time

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import TopKRecs, check_free, cuda_device, upload, upload_csr


def l1_rows(indptr, data):
    """fp32(v / sum |v|) per CSR row with the sum accumulated in fp64 in stored order, as sklearn's l1 `normalize`
    computes it; rows that sum to 0 are left alone.  Rows are walked position by position, longest first, so the work is
    O(nnz) numpy operations in max-row-length steps."""
    lens = np.diff(indptr)
    order = np.argsort(-lens, kind="stable")
    sl, start = lens[order], indptr[:-1][order]
    a = np.abs(data.astype(np.float64))
    s = np.zeros(len(order))
    for p in range(int(sl[0]) if len(sl) else 0):
        m = int(np.searchsorted(-sl, -p, side="left"))          # rows longer than p
        s[:m] += a[start[:m] + p]
    row_sum = np.empty(len(order))
    row_sum[order] = s
    per = np.repeat(row_sum, lens)
    out = data.astype(np.float32, copy=True)
    ok = per != 0.0
    out[ok] = (data[ok].astype(np.float64) / per[ok]).astype(np.float32)
    return out


class RP3Model:
    """W (a CSR on the device) and its scoring."""

    def __init__(self, data, neighborhood, alpha, beta, normalize_similarity, device):
        self.device = torch.device(device)
        self.R = data.sp_i_train_ratings.tocsr()
        self.n_users, self.n_items = self.R.shape
        self.k = self.n_items if neighborhood == -1 else int(neighborhood)
        if self.k < 1:
            raise ValueError(f"neighborhood={neighborhood}: a positive number of neighbours or -1 (every item)")
        self.alpha, self.beta, self.normalize = float(alpha), float(beta), bool(normalize_similarity)
        if self.R.nnz and float(self.R.data.min()) < 0:
            raise ValueError("RP3beta needs nonnegative ratings: its transition probabilities are ratings over row sums")
        self.urm = upload_csr(self.R.indptr, self.R.indices, self.R.data, self.device)
        self.W = None

    def host_operands(self):
        """(Pui with rows sorted by column, Piu, degree) as numpy CSR parts, computed as rp3beta.py:77-96 does."""
        R = self.R
        pui = l1_rows(R.indptr, R.data)
        count = np.bincount(R.indices, minlength=self.n_items)
        degree = np.zeros(self.n_items)
        nz = count != 0
        degree[nz] = np.power(count[nz].astype(np.float32), -self.beta)
        C = R.tocsc()
        C.sort_indices()                                     # Piu's rows list users ascending
        piu = np.repeat((1.0 / np.maximum(count, 1)).astype(np.float32), count)
        if self.alpha != 1.0:
            pui = np.power(pui, self.alpha)
            piu = np.power(piu, self.alpha)
        P = type(R)((pui, R.indices, R.indptr), shape=R.shape)
        P = P.sorted_indices()                               # per-column order depends only on Piu's user order
        return (P.indptr, P.indices, P.data), (C.indptr, C.indices, piu), degree

    def working_set(self, nnz_r):
        """(bytes needed at the peak, a description)."""
        n, kk = self.n_items, min(self.k, self.n_items)
        lists = n * kk * 8 + n * 4
        prune = n * kk * 9 + n * 16
        operands = 2 * (nnz_r * 8 + (max(n, self.n_users) + 1) * 8)
        rows = ops.rp3_row_workspace_bytes(n)
        g = 2 ** 30
        return lists + prune + operands + rows, (f"the similarity lists {lists / g:.1f} GiB ({n} x {kk} entries), the "
                                                 f"column prune {prune / g:.1f} GiB, the operands {operands / g:.1f} GiB")

    def initialize(self, mark=None):
        """W.  `mark(phase)`, when given, is called as each phase's work has been queued (host_prepare, upload,
        similarity, normalize when it runs, prune), so that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        self.W = None
        check_free("RP3beta", self.device, *self.working_set(self.R.nnz))
        pui, piu, degree = self.host_operands()
        # longest rows first: row i costs sum over its users of their rating counts
        work = np.bincount(self.R.indices, weights=np.diff(self.R.indptr)[np.repeat(np.arange(self.n_users),
                                                                                    np.diff(self.R.indptr))],
                           minlength=self.n_items)
        order = np.argsort(-work, kind="stable")
        mark("host_prepare")
        Pui, Piu = upload_csr(*pui, self.device), upload_csr(*piu, self.device)
        deg, order = upload(degree, self.device, torch.float64), upload(order, self.device, torch.int32)
        mark("upload")
        idx, val, cnt = ops.rp3_similarity(Piu, Pui, deg, self.k, order=order)
        mark("similarity")
        del Pui, Piu
        if self.normalize:
            ops.rp3_l1_rows(val, cnt)
            mark("normalize")
        self.W = ops.rp3_prune_cols(idx, val, cnt, self.k)
        mark("prune")

    def topk(self, k, mask_indptr, mask_indices, users=None, user_begin=0, n_sel=None):
        return sparse_score_topk(self.urm, self.W, self.n_items, k, mask_indptr, mask_indices, users, user_begin, n_sel)


def sparse_score_topk(urm, W, n_items, k, mask_indptr, mask_indices, users=None, user_begin=0, n_sel=None):
    """The masked top k of urm . W (both CSRs on the device) in SciPy's float32 csr * csr order, the selected rows
    visited longest first."""
    ap, ai, _ = urm
    rows = users.long() if users is not None else \
        torch.arange(user_begin, user_begin + (ap.numel() - 1 - user_begin if n_sel is None else n_sel), device=ap.device)
    # longest rows first: row u costs the lengths of the W rows its ratings select
    wl = torch.diff(W[0])
    cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=ap.device), torch.cumsum(wl[ai.long()], 0)])
    work = cs[ap[rows + 1]] - cs[ap[rows]]
    order = torch.argsort(work, descending=True, stable=True).to(torch.int32)
    return ops.rp3_score_topk(urm, W, n_items, k, mask_indptr, mask_indices, users=users, user_begin=user_begin,
                              n_sel=n_sel, order=order)


class RP3beta(TopKRecs, RecMixin, BaseRecommenderModel):
    r"""Updatable, accurate, diverse, and scalable recommendations for interactive applications
    (https://dl.acm.org/doi/10.1145/2955101), on the H100.  YAML block as the reference's: RP3beta: {meta: {...},
    neighborhood, alpha, beta, normalize_similarity}; optional keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_neighborhood", "neighborhood", "neighborhood", 10, int, None),
            ("_alpha", "alpha", "alpha", 1., float, None),
            ("_beta", "beta", "beta", 0.6, float, None),
            ("_normalize_similarity", "normalize_similarity", "normalize_similarity", False, bool, None)
        ]
        self.autoset_params()
        if self._neighborhood == -1:
            self._neighborhood = self._data.num_items
        if self._save_weights or self._restore:
            raise NotImplementedError("meta.save_weights / meta.restore are not supported for RP3beta: the reference "
                                      "pickles the dense prediction matrix, which this build never forms")
        self._device = cuda_device(self._params, "RP3beta")
        self._model = RP3Model(self._data, self._neighborhood, self._alpha, self._beta, self._normalize_similarity,
                               self._device)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)

    @property
    def name(self):
        return f"RP3beta_{self.get_params_shortcut()}"

    def train(self):
        start = time.time()
        self._model.initialize()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The similarity computation has taken: {time.time() - start}")
        self.evaluate()
