"""Evaluator for the host mirror: nDCG / HR / Precision / Recall with the reference's definitions
(elliot/evaluation/evaluator.py:79-147; ndcg.py:68-125; relevance.py:55,80-82; hit_rate.py, precision.py, recall.py),
and 19 more of the reference's list metrics (METRICS below: ranking accuracy, novelty, popularity bias, coverage and
diversity), vectorised over (users x k) index arrays.  tests/test_host_parity.py and tests/test_metrics_host.py check
them against numbers the reference's own Evaluator produced on the same lists (tests/golden).  AUC and GAUC rank every
relevant item in the whole catalogue: they come from the model's rank pass (ops.score_rank, counts per user) through
finish_auc, not from the lists, and are the same at every cutoff (tests/test_oracle_auc.py).

`eval_tensors` is the device path (SURVEY.md §8f #1): the top-k index tensor written by the scoring kernels is
scored against the test set by `eb_eval_topk_f64` (the four above) and `eb_eval_metrics_f64` (the 19 others) without
ever becoming Python tuples; same definitions, same numbers (fp64; summation order differs, <= 1e-12 relative)."""
import math

import numpy as np

from .dataset import eval_csr_of, eval_users_of

SUPPORTED = {"ndcg": "nDCG", "hr": "HR", "precision": "Precision", "recall": "Recall"}
# result keys are the reference's name() values; each kernel runs only when one of its metrics is asked for
METRICS = ("nDCGRendle2020", "MRR", "MAP", "MAR", "F1", "LAUC", "NumRetrieved", "EPC", "EFD", "ARP", "APLT", "ACLT",
           "PopREO", "PopRSP", "ItemCoverage", "UserCoverage", "UserCoverageAtN", "Gini", "SEntropy")
_EXTENDED = {m.lower(): m for m in METRICS}
# metrics of the rank of each relevant item in the whole catalogue: from the model's rank pass (counts per user), not from
# the top-k lists, and the same at every cutoff; available to an evaluator built with rank_pass=True
RANK = ("AUC", "GAUC")
_RANKED = {m.lower(): m for m in RANK}
_WHY_NOT = {
    **dict.fromkeys(("auc", "gauc"), "it ranks every relevant item in the whole catalogue, which takes a model's rank pass "
                                     "(build the Evaluator with rank_pass=True and give eval() its rank_counts)"),
    **dict.fromkeys(("mae", "mse", "rmse"), "it needs the predicted scores and the test ratings, not a top-k list"),
    **dict.fromkeys(("dsc", "extendedf1", "extendedepc", "extendedefd", "extendedpopreo", "extendedpoprsp"),
                    "it is a complex metric with parameters"),
    **dict.fromkeys(("srecall", "biasdisparitybr", "biasdisparitybs", "biasdisparitybd", "usermadrating", "itemmadrating",
                     "usermadranking", "itemmadranking", "reo", "rsp"), "it needs side-information files"),
}
# slots of the fp64 vector eb_eval_metrics_f64 writes (include/elliot_b200.h); the host mirror fills the same vector
(S_NREL, S_RENDLE, S_MRR, S_MAP, S_MAR, S_F1, S_LAUC, S_NUMRET, S_EPC, S_EFD, S_REO_NUM_H, S_REO_NUM_T, S_REO_DEN_H,
 S_REO_DEN_T, S_NROWS, S_ARP, S_APLT, S_ACLT, S_RSP_NUM_H, S_RSP_NUM_T, S_RSP_DEN_H, S_RSP_DEN_T, S_UCOV, S_UCOV_N,
 S_FREE_NORM, S_EMPTY, S_ITEMCOV, S_GINI_S, S_SENTROPY) = range(29)
N_SLOTS = 29
PER_USER = ("nDCGRendle2020", "MRR", "MAP", "MAR", "F1", "LAUC", "NumRetrieved", "EPC", "EFD", "ARP", "APLT", "ACLT")


def metric_tables(data, cs, has_rows):
    """The per-split tables the 19 metrics read, built once with vectorised NumPy.  Per private user (user_info, int32
    n_users x 6): has any row in the split, |train_u| (lauc.py), PopREO denominators |(class & rel_u) - train_u| and
    PopRSP denominators |class - train_u| for class = short head, long tail (pop_reo.py, pop_rsp.py).  Per private
    item: pop (train users, popularity.py get_pop_items), long_tail (popularity.py: items walked in stable descending
    pop order fill the short head until 0.8 * transactions is used up, the item crossing the limit included), nov
    (EPC novelty 1 - pop/num_users, EFD novelty -log2(pop / sum pop); epc.py, efd.py)."""
    from types import SimpleNamespace
    m = data.sp_i_train.tocsr()
    n_users, n_items = m.shape
    pop = np.bincount(m.indices, minlength=n_items).astype(np.int64)
    order = np.argsort(-pop, kind="stable")
    crossed = np.flatnonzero(data.transactions * 0.8 - np.cumsum(pop[order]) <= 0)
    n_head = int(crossed[0]) + 1 if crossed.size else n_items
    long_tail = np.ones(n_items, np.uint8)
    long_tail[order[:n_head]] = 0
    with np.errstate(divide="ignore"):
        nov = np.stack([1 - pop / n_users, -np.log(pop / pop.sum()) / np.log(2)], 1)
    train_rows = np.repeat(np.arange(n_users, dtype=np.int64), np.diff(m.indptr))
    indptr, rel_idx, _ = cs
    rel_rows = np.repeat(np.arange(n_users, dtype=np.int64), np.diff(indptr))
    known = rel_idx >= 0                                             # test-only items are in neither class
    not_train = ~np.isin(rel_rows * n_items + rel_idx, train_rows * n_items + m.indices)
    rel_lt = long_tail[np.where(known, rel_idx, 0)]
    per_user = lambda rows, sel: np.bincount(rows[sel], minlength=n_users)
    train_lt = per_user(train_rows, long_tail[m.indices] == 1)
    n_train = np.diff(m.indptr)
    user_info = np.stack([has_rows, n_train,
                          per_user(rel_rows, known & not_train & (rel_lt == 0)),
                          per_user(rel_rows, known & not_train & (rel_lt == 1)),
                          (n_items - long_tail.sum()) - (n_train - train_lt),
                          long_tail.sum() - train_lt], 1).astype(np.int32)
    return SimpleNamespace(user_info=user_info, pop=pop, long_tail=long_tail, nov=nov, n_items=n_items)


def position_tables(k):
    """Per position r < k: discount ln2/ln(r+2) (relevance.py:55), MAP tail H(k) - H(r) = sum_{n=r+1..k} 1/n (a hit at r
    adds 1/n to P@n for every n > r, map.py); inv_idcg[m] = 1 / sum_{i<m} discount[i], the binary ideal DCG of a user
    with min(|rel|, k) = m (ndcg_rendle2020.py)."""
    disc = np.array([math.log(2) / math.log(r + 2) for r in range(k)])
    tail = np.cumsum(1.0 / np.arange(k, 0, -1))[::-1].copy()
    inv_idcg = np.zeros(k + 1)
    inv_idcg[1:] = 1.0 / np.cumsum(disc)
    return disc, tail, inv_idcg


def host_metric_sums(tab, cs, priv_users, idx, k, per_user=False):
    """The vector eb_eval_metrics_f64 computes, from a host (n, >=k) array of private item ids (-1 = end of the list)
    with rows aligned to priv_users; per_user=True also returns the (n x 12) PER_USER values, NaN where the reference
    has none."""
    indptr, rel_idx, _ = cs
    n_items = tab.n_items
    disc, tail, inv_idcg = position_tables(k)
    pu = np.asarray(priv_users, np.int64)
    L = np.asarray(idx)[:, :k].astype(np.int64)
    info = tab.user_info[pu].astype(np.int64)
    A = info[:, 0] != 0                                              # users with any test row
    valid = np.cumprod(L >= 0, axis=1).astype(bool) & A[:, None]     # the list: entries before the first -1
    n = valid.sum(1)
    nrel = np.where(A, indptr[pu + 1] - indptr[pu], 0)
    B = nrel > 0                                                     # ... and with a relevant item
    Li = np.where(valid, L, 0)
    rel_rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr))
    keep = rel_idx >= 0
    hit = valid & B[:, None] & np.isin(pu[:, None] * n_items + Li, rel_rows[keep] * n_items + rel_idx[keep])
    r = np.arange(k)
    h = hit.sum(1)
    sum_r = (hit * r).sum(1)
    nr = np.maximum(nrel, 1)
    m_rel = np.minimum(nr, k)
    neg = n_items - info[:, 1] - nrel + 1
    p, rc = h / k, h / nr
    den = p + rc
    norm = (valid * disc).sum(1)
    nz = np.where(norm > 0, norm, 1)
    lt = valid & (tab.long_tail[Li] == 1)
    n_lt = lt.sum(1)
    n1 = np.maximum(n, 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        user_b = np.stack([
            inv_idcg[m_rel] * (hit * disc).sum(1),                                 # nDCGRendle2020
            np.where(h > 0, 1.0 / (np.argmax(hit, 1) + 1), 0.0),                   # MRR
            (hit * tail).sum(1) / k,                                               # MAP
            (h * k - sum_r) / nr / k,                                              # MAR
            np.where(den != 0, 2 * p * rc / np.where(den != 0, den, 1), 0.0),      # F1
            (h * neg - sum_r + h * (h - 1) // 2) / neg / m_rel,                    # LAUC
            n.astype(np.float64),                                                  # NumRetrieved
            (hit * disc * tab.nov[Li, 0]).sum(1) / nz,                             # EPC
            (hit * disc * tab.nov[Li, 1]).sum(1) / nz], 1)                         # EFD
    user_a = np.stack([(valid * tab.pop[Li]).sum(1) / n1, n_lt / n1, n_lt.astype(np.float64)], 1)   # ARP APLT ACLT
    counts = np.bincount(L[valid], minlength=n_items)
    cs_sorted = np.sort(counts[counts > 0])
    free_norm = int(n[A].sum())
    with np.errstate(divide="ignore"):
        nov_s = -np.log(np.where(valid, counts[Li], 1) / max(free_norm, 1)) / np.log(2)
    s = np.zeros(N_SLOTS)
    hits_sh = (hit & ~lt).sum(1)
    s[S_NREL] = B.sum()
    s[S_RENDLE:S_EFD + 1] = user_b[B].sum(0)
    s[S_REO_NUM_H], s[S_REO_NUM_T] = hits_sh[B].sum(), (h - hits_sh)[B].sum()
    s[S_REO_DEN_H], s[S_REO_DEN_T] = info[B, 2].sum(), info[B, 3].sum()
    s[S_NROWS] = A.sum()
    s[S_ARP:S_ACLT + 1] = user_a[A].sum(0)
    s[S_RSP_NUM_H], s[S_RSP_NUM_T] = (n - n_lt)[A].sum(), n_lt[A].sum()
    s[S_RSP_DEN_H], s[S_RSP_DEN_T] = info[A, 4].sum(), info[A, 5].sum()
    s[S_UCOV], s[S_UCOV_N] = (n > 0)[A].sum(), (n >= k)[A].sum()
    s[S_FREE_NORM] = free_norm
    s[S_EMPTY] = (n == 0)[A].sum()
    s[S_ITEMCOV] = cs_sorted.size
    s[S_GINI_S] = int((np.arange(cs_sorted.size, dtype=np.int64) * cs_sorted).sum())
    s[S_SENTROPY] = ((valid * nov_s).sum(1)[n > 0] / n[n > 0]).sum()
    if not per_user:
        return s, None
    pv = np.full((len(pu), len(PER_USER)), np.nan)
    pv[B, :9] = user_b[B]
    ok = A & (n > 0)
    pv[ok, 9:11] = user_a[ok, :2]
    pv[A, 11] = user_a[A, 2]
    return s, pv


def finish_auc(n_pos, sum_c, n_rel, n_train, n_items, names):
    """AUC and GAUC (auc.py, gauc.py) from the rank pass's per-user counts (ops.score_rank): n_pos relevant items in the
    user's full list and sum_c, the sum over them of the non-relevant entries ahead of each.  With neg_u = n_items -
    |train_u| - |R_u| + 1 each such item's term is (neg_u - c_i) / neg_u, so a user's terms sum to
    (n_pos neg_u - sum_c) / neg_u.  AUC is the mean of every term of the users with |R_u| > 0, GAUC the mean over those
    users of their sum / |R_u|; like np.average([]), no term (or no user) gives NaN, and neg_u = 0 under a term raises
    ZeroDivisionError, as the reference's int / int does."""
    n_pos, sum_c, n_rel, n_train = (np.asarray(a, np.int64) for a in (n_pos, sum_c, n_rel, n_train))
    B = n_rel > 0
    neg = n_items - n_train - n_rel + 1
    if (B & (n_pos > 0) & (neg == 0)).any():
        raise ZeroDivisionError("AUC/GAUC: a user with a ranked relevant item has no negative item (neg_num = 0)")
    with np.errstate(divide="ignore", invalid="ignore"):
        user_sum = np.where(n_pos > 0, (n_pos * neg - sum_c) / np.where(neg != 0, neg, 1), 0.0)[B]
    n_terms, n_users = int(n_pos[B].sum()), int(B.sum())
    out = {"AUC": float(user_sum.sum() / n_terms) if n_terms else float("nan"),
           "GAUC": float((user_sum / n_rel[B]).sum() / n_users) if n_users else float("nan")}
    return {m: out[m] for m in names}


def finish_metrics(s, k, n_items, names):
    """Metric values from the slot vector: means over the users each metric averages over (0.0 when there are none,
    like the four accuracy metrics), the ratios of PopREO / PopRSP and the closed forms of Gini and SEntropy."""
    s = np.asarray(s, np.float64)
    n_rel, n_rows = s[S_NREL], s[S_NROWS]
    if ("ARP" in names or "APLT" in names) and s[S_EMPTY] > 0:
        raise ZeroDivisionError(f"ARP/APLT: {int(s[S_EMPTY])} user(s) with test rows have an empty recommendation list")

    def ratio(num, den):                                             # np.std(pr) / np.mean(pr) of pop_reo.py / pop_rsp.py
        with np.errstate(divide="ignore", invalid="ignore"):
            pr = np.array(num) / np.array(den)
            return float(np.std(pr) / np.mean(pr))
    out = {}
    for m in names:
        if m in PER_USER[:9]:
            out[m] = float(s[S_RENDLE + PER_USER.index(m)] / n_rel) if n_rel else 0.0
        elif m in ("ARP", "APLT", "ACLT"):
            out[m] = float(s[S_ARP + PER_USER.index(m) - 9] / n_rows) if n_rows else 0.0
        elif m == "PopREO":
            out[m] = ratio(s[[S_REO_NUM_H, S_REO_NUM_T]], s[[S_REO_DEN_H, S_REO_DEN_T]]) if n_rel else 0.0
        elif m == "PopRSP":
            out[m] = ratio(s[[S_RSP_NUM_H, S_RSP_NUM_T]], s[[S_RSP_DEN_H, S_RSP_DEN_T]]) if n_rows else 0.0
        elif m == "ItemCoverage":
            out[m] = int(s[S_ITEMCOV])
        elif m == "UserCoverage":
            out[m] = int(s[S_UCOV])
        elif m == "UserCoverageAtN":
            out[m] = int(s[S_UCOV_N])
        elif m == "Gini":
            # gini_index.py: 1 - sum_j (2 (j + N - n + 1) - N - 1) cs_j / F / (N - 1) = 1 - (2 S / F + N - 2 n + 1) / (N - 1)
            F, n = s[S_FREE_NORM], s[S_ITEMCOV]
            out[m] = float(1 - ((2 * s[S_GINI_S] / F + n_items - 2 * n + 1) if F else 0.0) / (n_items - 1)) if n_rows else 0.0
        elif m == "SEntropy":
            out[m] = float(s[S_SENTROPY] / n_rows) if n_rows else 0.0
    return out


class Evaluator:
    def __init__(self, data, params, rank_pass=False):
        """rank_pass: the caller supplies rank_counts (a model's ops.score_rank counts) to eval() / eval_tensors(), so
        AUC and GAUC are available; without it they raise here, like every other name this evaluator cannot compute."""
        self._data, self._params = data, params
        ev = data.config.evaluation
        self._k = getattr(ev, "cutoffs", [data.config.top_k])
        self._k = self._k if isinstance(self._k, list) else [self._k]
        if any(np.array(self._k) > data.config.top_k):
            raise Exception("Cutoff values must be smaller than recommendation list length (top_k)")
        self._metrics = []
        for m in ev.simple_metrics:
            name = SUPPORTED.get(m.lower()) or _EXTENDED.get(m.lower()) or (_RANKED.get(m.lower()) if rank_pass else None)
            if name is None:
                why = _WHY_NOT.get(m.lower(), "the reference does not know this name")
                raise Exception(f"metric {m} is not available in elliot_b200's evaluator: {why} "
                                f"(use the reference Evaluator through ProxyRecommender)")
            self._metrics.append(name)
        self._basic = [m for m in self._metrics if m in SUPPORTED.values()]
        self._extended = [m for m in self._metrics if m in METRICS]
        self._ranked = [m for m in self._metrics if m in RANK]
        self._sets = {"test": eval_csr_of(data, "test"), "val": eval_csr_of(data, "val")}

    def get_needed_recommendations(self):
        return self._data.config.top_k

    @property
    def needs_rank(self):
        """True when AUC or GAUC is asked for: evaluate() then runs the model's rank pass once per split
        (rank_sets / rank_counts) besides its top-k lists."""
        return bool(self._ranked)

    def rank_sets(self, device):
        """{split: (rel indptr int64, item-sorted rel items int32)} on `device` for every split that exists: the
        arguments of a model's rank pass."""
        return {w: self._device_set(w, self._k[0], device)[:2] for w in ("val", "test") if self._sets[w] is not None}

    def _rank_values(self, which, rank_counts):
        """AUC / GAUC of a split from the host (n_pos, sum_c) arrays of its rank pass (rows = private users)."""
        if not self._ranked:
            return {}
        if rank_counts is None:
            raise Exception(f"{'/'.join(self._ranked)} need the model's rank pass counts (rank_counts)")
        n_train = np.diff(self._data.sp_i_train.tocsr().indptr)
        return finish_auc(*rank_counts[which], np.diff(self._sets[which][0]), n_train, self._data.num_items, self._ranked)

    # recommendations: (val, test) pair of {public_user: [(public_item, score), ...]}
    # rank_counts: {split: (n_pos, sum_c)} host arrays of the model's rank pass, when AUC or GAUC is asked for
    def eval(self, recommendations, rank_counts=None):
        out = {}
        ranked = {w: self._rank_values(w, rank_counts) for w in ("val", "test") if self._sets[w] is not None}
        for k in self._k:
            res = {}
            for slot, which in ((0, "val"), (1, "test")):
                cs = self._sets[which]
                res[which] = None if cs is None else self._eval_dict(recommendations[slot], which, k, ranked[which])
            if res["val"] is None:
                res["val"] = res["test"]
            if res["test"] is None:
                res["test"] = res["val"]
            out[k] = {"val_results": res["val"], "val_statistical_results": {},
                      "test_results": res["test"], "test_statistical_results": {}}
        return out

    def _tables(self, which):
        """metric_tables of the split (cached); None when the split does not exist."""
        cache = self.__dict__.setdefault("_metric_tables", {})
        if which not in cache:
            cs = self._sets[which]
            cache[which] = None if cs is None else metric_tables(self._data, cs, eval_users_of(self._data, which))
        return cache[which]

    # ---- device path ---------------------------------------------------------------------------
    def _device_set(self, which, k, device):
        """Item-sorted relevant-item CSR + per-user IDCG@k + discounts on `device` (cached)."""
        import torch
        key = (which, k, str(device))
        cache = self.__dict__.setdefault("_dev_sets", {})
        if key in cache:
            return cache[key]
        cs = self._sets[which]
        if cs is None:
            cache[key] = None
            return None
        indptr, idx, gain = cs
        n = len(indptr) - 1
        rows = np.repeat(np.arange(n), np.diff(indptr))
        disc = np.array([math.log(2) / math.log(r + 2) for r in range(k)])      # relevance.py:55
        by_gain = np.lexsort((-gain, rows))                                      # ideal ranking per user
        rank = np.arange(len(rows)) - indptr[rows]
        top = rank < k
        idcg = np.bincount(rows[top], weights=gain[by_gain][top] * disc[rank[top]], minlength=n)
        by_item = np.lexsort((idx, rows))                                        # lookup rows sorted by item id
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dt)
        cache[key] = (t(indptr, torch.int64), t(idx[by_item], torch.int32), t(gain[by_item], torch.float64),
                      t(idcg, torch.float64), t(disc, torch.float64))
        return cache[key]

    def _metric_device_set(self, which, k, device):
        """The arguments of ops.eval_topk_metrics after k, on `device` (cached per split, k and device)."""
        import torch
        key = (which, k, str(device))
        cache = self.__dict__.setdefault("_metric_dev_sets", {})
        if key not in cache:
            ds, tab = self._device_set(which, k, device), self._tables(which)
            t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dt)
            cache[key] = (ds[0], ds[1], t(tab.user_info, torch.int32), t(tab.pop, torch.int32),
                          t(tab.long_tail, torch.uint8), t(tab.nov, torch.float64),
                          *(t(a, torch.float64) for a in position_tables(k)))
        return cache[key]

    def eval_tensors(self, idx, users=None, rank_counts=None):
        """Same result structure as eval(), from a device (rows x top_k) int32 tensor of PRIVATE item ids
        (-1 = empty), row r = private user r (or users[r])."""
        from . import ops
        out = {}
        ranked = {w: self._rank_values(w, rank_counts) for w in ("val", "test") if self._sets[w] is not None}
        for k in self._k:
            res = {}
            for which in ("val", "test"):
                ds = self._device_set(which, k, idx.device)
                if ds is None:
                    res[which] = None
                    continue
                vals = dict(ranked[which])
                if self._basic:
                    sums, _ = ops.eval_topk(idx, k, *ds, users=users)
                    sums = sums.cpu().numpy()
                    n = sums[0]
                    vals.update(zip(("nDCG", "HR", "Precision", "Recall"), (sums[1:] / n if n else np.zeros(4)).tolist()))
                if self._extended:
                    s, _ = ops.eval_topk_metrics(idx, k, *self._metric_device_set(which, k, idx.device), users=users)
                    vals.update(finish_metrics(s.cpu().numpy(), k, self._tables(which).n_items, self._extended))
                res[which] = {m: vals[m] for m in self._metrics}
            if res["val"] is None:
                res["val"] = res["test"]
            if res["test"] is None:
                res["test"] = res["val"]
            out[k] = {"val_results": res["val"], "val_statistical_results": {},
                      "test_results": res["test"], "test_statistical_results": {}}
        return out

    def _eval_dict(self, recs, which, k, ranked):
        pub_u, pub_i = self._data.public_users, self._data.public_items
        users = [u for u in recs if u in pub_u]
        idx = np.full((len(users), k), -1, np.int64)
        for r, u in enumerate(users):
            row = [pub_i.get(it, -1) for it, _ in recs[u][:k]]
            idx[r, :len(row)] = row
        priv = np.array([pub_u[u] for u in users], np.int64)
        vals = self.eval_arrays(priv, idx, self._sets[which], k) if self._basic else {}
        if self._extended:
            tab = self._tables(which)
            s, _ = host_metric_sums(tab, self._sets[which], priv, idx, k)
            vals.update(finish_metrics(s, k, tab.n_items, self._extended))
        vals.update(ranked)
        return {m: vals[m] for m in self._metrics}

    def eval_arrays(self, priv_users, idx, cs, k):
        """idx: (n, >=k) private item ids (−1 = empty slot), rows aligned with priv_users."""
        indptr, rel_idx, rel_gain = cs
        disc = np.array([math.log(2) / math.log(r + 2) for r in range(k)])      # relevance.py:55
        acc = {m: [] for m in self._basic}
        for row, pu in zip(idx[:, :k], priv_users):
            lo, hi = indptr[pu], indptr[pu + 1]
            if hi == lo:                       # users without relevant test items are skipped
                continue
            gains = dict(zip(rel_idx[lo:hi].tolist(), rel_gain[lo:hi].tolist()))
            g = np.array([gains.get(int(it), 0.0) if it >= 0 else 0.0 for it in row])
            hits = g > 0
            if "nDCG" in acc:
                ideal = np.sort(rel_gain[lo:hi])[::-1][:k]
                idcg = float((ideal * disc[:len(ideal)]).sum())
                dcg = float((g * disc[:len(g)]).sum())
                acc["nDCG"].append(dcg / idcg if dcg > 0 else 0.0)
            if "HR" in acc:
                acc["HR"].append(1.0 if hits.any() else 0.0)
            # Precision/Recall sum the DISCOUNTED-relevance lookups? No: binary relevance
            # (precision.py / recall.py use relevance.binary_relevance.get_rel -> 1/0).
            if "Precision" in acc:
                acc["Precision"].append(hits.sum() / k)
            if "Recall" in acc:
                acc["Recall"].append(hits.sum() / (hi - lo))
        return {m: (float(np.mean(v)) if v else 0.0) for m, v in acc.items()}
