"""The reference's clustered fairness metrics (elliot/evaluation/metrics/fairness): BiasDisparityBR / BS / BD,
User/ItemMADrating, User/ItemMADranking, REO and RSP, asked for as `evaluation.complex_metrics` entries that name a
clustering file of users or items.

A clustering file is `id<TAB>cluster` per line with public ids, read as the reference reads it (pandas, header=None).
Labels must be the integers 0..n-1, n the number of distinct labels, and an id may appear once; anything else is
refused when the Evaluator is built (the reference fails late, wraps negative labels, or keeps the last label of a
repeated id in some metrics and every label in others).  An entry without a file behaves as the reference does: one
cluster and an empty mapping, so BiasDisparity puts every user and item in group 0, MAD skips every user or item and
REO / RSP count nothing (0 / 0).

One pass over the lists (eb_eval_fairness_f64 on the device, host_fairness_sums here) fills one vector of counts and
one of sums per (user clustering, item clustering) pair; finish() turns them into the reference's values with its NumPy
arithmetic.  BiasDisparityBS (the train matrix alone) and the REO / RSP denominators are integers computed here."""
import os
import warnings
from types import SimpleNamespace

import numpy as np
import pandas as pd

COMPLEX = ("BiasDisparityBR", "BiasDisparityBS", "BiasDisparityBD", "UserMADrating", "ItemMADrating", "UserMADranking",
           "ItemMADranking", "REO", "RSP")
_BY_LOWER = {m.lower(): m for m in COMPLEX}
_WHY_NOT = {
    **dict.fromkeys(("dsc", "extendedf1", "extendedepc", "extendedefd", "extendedpopreo", "extendedpoprsp"),
                    "the evaluator's complex metrics are the clustered fairness metrics only"),
    "srecall": "it needs an item feature file",
}


def _why_not(name):
    return _WHY_NOT.get(name.lower(), "the reference does not know this name")


# ---- clustering files ---------------------------------------------------------------------------------------------
_FILES = {}


def read_clustering(path):
    """The file's ids and labels (cached per absolute path and modification time), with n = the number of clusters and sizes[c] = the ids
    of cluster c over the whole file, ids absent from the dataset included.  Raises ValueError on labels that are
    not 0..n-1 and on repeated ids."""
    path = os.path.abspath(path)
    st = os.stat(path)
    key = (path, st.st_mtime_ns, st.st_size)
    if key not in _FILES:
        df = pd.read_csv(path, sep="\t", header=None)
        if df.shape[1] < 2:
            raise ValueError(f"clustering file {path}: expected id<TAB>cluster lines")
        ids, labels = df[0].to_numpy(), df[1].to_numpy()
        n = int(pd.Series(labels).nunique())
        if not np.issubdtype(labels.dtype, np.integer) or not np.array_equal(np.unique(labels), np.arange(n)):
            raise ValueError(f"clustering file {path}: the labels must be the integers 0..{n - 1} ({n} distinct labels), "
                             f"got {np.unique(labels)[:8].tolist()}")
        dup = pd.Index(ids).duplicated()
        if dup.any():
            raise ValueError(f"clustering file {path}: id {ids[dup][0]!r} is listed more than once")
        labels = labels.astype(np.int64)
        _FILES[key] = SimpleNamespace(path=path, ids=ids, labels=labels, n=n, sizes=np.bincount(labels, minlength=n))
    return _FILES[key]


def private_labels(cl, public_ids, default):
    """int32 cluster of each private id (public_ids[private]): the file's label, -1 when the file does not list it;
    without a file (cl None) every id gets `default`."""
    if cl is None:
        return np.full(len(public_ids), default, np.int32)
    pos = pd.Index(cl.ids).get_indexer(pd.Index(public_ids))
    return np.where(pos >= 0, cl.labels[np.maximum(pos, 0)], -1).astype(np.int32)


# ---- entries ------------------------------------------------------------------------------------------------------
class Entry:
    """One complex_metrics entry: the metric, its clusterings and its result keys (the reference's get() names)."""

    def __init__(self, spec):
        if not isinstance(spec, dict) or "metric" not in spec:
            raise Exception(f"complex metric entry {spec!r} has no `metric` key")
        m = str(spec["metric"])
        self.metric = _BY_LOWER.get(m.lower())
        if self.metric is None:
            raise Exception(f"metric {m} is not available in elliot_b200's evaluator: {_why_not(m)} "
                            f"(use the reference Evaluator through ProxyRecommender)")

        def load(file_key, name_key, name_required=True):
            path = spec.get(file_key)
            if not path:
                return None, ""
            if name_required and name_key not in spec:
                raise Exception(f"{self.metric}: `{file_key}` needs `{name_key}`")
            try:
                return read_clustering(path), str(spec.get(name_key, ""))
            except ValueError as ex:
                raise Exception(f"{self.metric}: {ex}") from None
        if self.metric.startswith("BiasDisparity"):
            self.users, self.uname = load("user_clustering_file", "user_clustering_name")
            self.items, self.iname = load("item_clustering_file", "item_clustering_name")
            self.udefault = self.idefault = 0                    # no file: everyone in group 0
        else:
            mad = "MAD" in self.metric                             # MAD reads its name with a "" default
            cl, name = load("clustering_file", "clustering_name", name_required=not mad)
            if mad:
                name = str(spec.get("clustering_name", ""))
            if self.metric.startswith("User"):
                self.users, self.uname, self.items, self.iname = cl, name, None, ""
            else:
                self.users, self.uname, self.items, self.iname = None, "", cl, name
            self.udefault = self.idefault = -1                   # no file: nobody is clustered
        self.nu = self.users.n if self.users is not None else 1
        self.ni = self.items.n if self.items is not None else 1

    @property
    def launch(self):
        """Entries with the same key share one pass over the lists."""
        return (self.users and self.users.path, self.udefault, self.items and self.items.path, self.idefault)

    @property
    def needs_scores(self):
        return self.metric.endswith("MADrating")

    def keys(self):
        m = self.metric
        if "MAD" in m:
            return [f"{m}_{self.uname if m.startswith('User') else self.iname}"]
        if m.startswith("BiasDisparity"):
            return [f"{m}_users:{self.uname}-{g}_items:{self.iname}-{c}" for g in range(self.nu) for c in range(self.ni)]
        return [f"{m}-ProbToBeRanked_items:{self.iname}-{c}" for c in range(self.ni)] + [f"{m}_items:{self.iname}"]


# ---- the pass over the lists --------------------------------------------------------------------------------------
def layout(nu, ni):
    """Slices of the counts and sums vectors (include/elliot_b200.h, eb_eval_fairness_f64)."""
    o = nu + nu * ni
    return SimpleNamespace(users=slice(0, nu), br=slice(nu, o), reo=slice(o, o + ni), rsp=slice(o + ni, o + 2 * ni),
                           items=slice(o + 2 * ni, o + 3 * ni), ndcg=slice(0, nu), mean=slice(nu, 2 * nu),
                           irank=slice(2 * nu, 2 * nu + ni), irate=slice(2 * nu + ni, 2 * nu + 2 * ni))


def host_fairness_sums(priv_users, idx, scores, k, cs, idcg, has_rows, ucl, nu, icl, ni):
    """The (counts int64, sums fp64) eb_eval_fairness_f64 computes, from a host (n, >=k) array of private item ids
    (-1 ends a list) with rows aligned to priv_users and their scores (None: the rating sums are 0)."""
    indptr, rel_idx, rel_gain = cs
    n_items = len(icl)
    pu = np.asarray(priv_users, np.int64)
    L = np.asarray(idx)[:, :k].astype(np.int64)
    S = np.zeros(L.shape) if scores is None else np.asarray(scores, np.float64)[:, :k]
    A = np.asarray(has_rows, bool)[pu]
    valid = np.cumprod(L >= 0, axis=1).astype(bool) & A[:, None]
    n = valid.sum(1)
    B = A & (indptr[pu + 1] - indptr[pu] > 0)
    Li = np.where(valid, L, 0)
    rel_rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr))
    keep = rel_idx >= 0
    key = rel_rows[keep] * n_items + rel_idx[keep]
    order = np.argsort(key, kind="stable")
    key, g_rel = key[order], rel_gain[keep][order]
    q = pu[:, None] * n_items + Li
    pos = np.minimum(np.searchsorted(key, q), max(len(key) - 1, 0))
    hit = valid & B[:, None] & (key[pos] == q if len(key) else False)
    gain = np.where(hit, g_rel[pos] if len(key) else 0.0, 0.0)
    disc = np.log(2) / np.log(np.arange(k) + 2.0)
    dcg = (gain * disc).sum(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        ndcg = np.where(dcg > 0, dcg / np.where(dcg > 0, idcg[pu], 1), 0.0)
        mean = (S * valid).sum(1) / n if scores is not None else np.zeros(len(pu))
    gu = np.asarray(ucl)[pu]
    ci = np.asarray(icl)[Li]
    first = valid & ~np.tril(Li[:, :, None] == Li[:, None, :], -1).any(2)
    L_ = layout(nu, ni)
    counts = np.zeros(nu + nu * ni + 3 * ni, np.int64)
    sums = np.zeros(2 * nu + 2 * ni)
    su = B & (gu >= 0)
    counts[L_.users] = np.bincount(gu[su], minlength=nu)
    sums[L_.ndcg] = np.bincount(gu[su], weights=ndcg[su], minlength=nu)
    sums[L_.mean] = np.bincount(gu[su], weights=mean[su], minlength=nu)
    br = valid & (gu[:, None] >= 0) & (ci >= 0)
    counts[L_.br] = np.bincount((np.broadcast_to(gu[:, None], L.shape) * ni + ci)[br], minlength=nu * ni)
    counts[L_.reo] = np.bincount(ci[first & hit & (ci >= 0)], minlength=ni)
    counts[L_.rsp] = np.bincount(ci[first & (ci >= 0)], minlength=ni)
    ent = valid & B[:, None]                                     # row order, then position order
    e_it = Li[ent]
    cnt = np.bincount(e_it, minlength=n_items)
    gs, rs = np.zeros(n_items), np.zeros(n_items)
    np.add.at(gs, e_it, gain[ent])                               # applied in entry order: the reference's dict walk
    np.add.at(rs, e_it, np.where(hit, S, 0.0)[ent])
    listed = np.flatnonzero((cnt > 0) & (np.asarray(icl) >= 0))
    c_of = np.asarray(icl)[listed]
    counts[L_.items] = np.bincount(c_of, minlength=ni)
    sums[L_.irank] = np.bincount(c_of, weights=gs[listed] / cnt[listed], minlength=ni)
    sums[L_.irate] = np.bincount(c_of, weights=rs[listed] / cnt[listed], minlength=ni)
    return counts, sums


# ---- host tables and the finish -----------------------------------------------------------------------------------
def relevant_public(data, which):
    """(private user, public item, private item or -1) of the split's relevant rows (rating >= threshold)."""
    thr = data.config.evaluation.relevance_threshold
    if hasattr(data, "eval_arrays"):
        arr = data.eval_arrays(which, public=True)
        if arr is None:
            return None
        pu, pi, r, pub = arr
        keep = r >= thr
        return pu[keep], pub[keep], pi[keep]
    d = data.test_dict if which == "test" else getattr(data, "val_dict", None)
    if d is None:
        return None
    rows = [(pu, it, data.public_items.get(it, -1)) for pu, u in enumerate(data.users)
            for it, s in d.get(u, {}).items() if s >= thr]
    if not rows:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64)
    pu, pub, pi = zip(*rows)
    return np.array(pu, np.int64), np.array(pub), np.array(pi, np.int64)


def bias_source(data, ucl, nu, icl, ni, pc):
    """BiasDisparityBS: the train entries per (user cluster, item cluster), normalised like BiasDisparityBR."""
    m = data.sp_i_train.tocsr()
    rows = np.repeat(np.arange(m.shape[0]), np.diff(m.indptr))
    gu, ci = ucl[rows], icl[m.indices]
    ok = (gu >= 0) & (ci >= 0)
    cat = np.bincount(gu[ok] * ni + ci[ok], minlength=nu * ni).reshape(nu, ni).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return ((cat.T / cat.sum(1)).T) / pc


def _mad(s, n):
    """The reference's MAD: per-cluster averages sum / n, then the mean absolute difference over every pair of clusters
    (np.average([]) = NaN for a single cluster)."""
    n = np.asarray(n, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        avg = [s[i] / n[i] for i in range(len(s))]
        differences = [abs(avg[i] - avg[j]) for i in range(len(s)) for j in range(i + 1, len(s))]
        return float(np.average(differences))


def _parity(num, den):
    with np.errstate(divide="ignore", invalid="ignore"):
        pr = np.asarray(num, np.float64) / np.asarray(den, np.float64)
        return pr, np.std(pr) / np.mean(pr)


def finish(entry, counts, sums, bs=None, pc=None, den=None):
    """{result key: value} of one entry from its pass's vectors; bs = its BiasDisparityBS matrix, pc = the item
    clusters' share of the item file, den = the REO or RSP denominators."""
    m, nu, ni = entry.metric, entry.nu, entry.ni
    L_ = layout(nu, ni)
    counts, sums = np.asarray(counts), np.asarray(sums, np.float64)
    if m == "UserMADranking":
        vals = [_mad(sums[L_.ndcg], counts[L_.users])]
    elif m == "UserMADrating":
        vals = [_mad(sums[L_.mean], counts[L_.users])]
    elif m == "ItemMADranking":
        vals = [_mad(sums[L_.irank], counts[L_.items])]
    elif m == "ItemMADrating":
        vals = [_mad(sums[L_.irate], counts[L_.items])]
    elif m == "BiasDisparityBS":
        vals = bs.ravel().tolist()
    elif m in ("BiasDisparityBR", "BiasDisparityBD"):
        cat = counts[L_.br].reshape(nu, ni).astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            br = ((cat.T / cat.sum(1)).T) / pc
            vals = (br if m == "BiasDisparityBR" else (br - bs) / bs).ravel().tolist()
    else:
        pr, overall = _parity(counts[L_.reo if m == "REO" else L_.rsp], den)
        vals = pr.tolist() + [overall]
    return dict(zip(entry.keys(), (float(v) for v in vals)))
