"""DataSet mirror: the fields of elliot/dataset/dataset.py:177-245 that the hot path consumes,
with the reference's id ordering (users in first-appearance order; private item index =
iteration order of a CPython set, dataset.py:201-202), plus the CSR tensors the kernels read.

Out of scope (SURVEY.md §2 #3, #4, #8-#10): side information, prefiltering, eval-time negative
sampling.  The dense `allunrated_mask` (dataset.py:245) is available lazily for code that wants
it; the kernels mask through the train CSR instead (a dense mask is 40 TB at C5 scale)."""
import logging
from types import SimpleNamespace

import numpy as np
import pandas as pd
import scipy.sparse as sp


class DataSet:
    """Sort-based build (SURVEY.md §8f #2): everything the kernels need — id maps, the train CSR, the relevant-item CSR of
    the test/validation split — comes from factorize / stable argsort / scipy COO->CSR over the frame's columns; no
    per-row or per-user Python.  The reference's own build (`dataframe_to_dict`, dataset.py:247-255) filters the frame
    once per user, O(U*N).  The dict-of-dicts views the reference API exposes (`train_dict`, `i_train_dict`,
    `test_dict`, `val_dict`) are materialised lazily, only if something asks for them (the host evaluator, the exact
    sampler's set-order rows); the throughput path never does.

    Orderings are the reference's: users in first-appearance order; `items = list({k for a in train_dict.values() for k
    in a})` (dataset.py:201-202) — a CPython set filled in (user first-appearance, row) order, reproduced by inserting
    the items' first occurrences in exactly that order into a real `set`; duplicate (user, item) rows keep their first
    position and their last rating, like the dict they came from."""

    def __init__(self, config, data_tuple, *args, **kwargs):
        self.logger = logging.getLogger("elliot_b200.DataSet")
        self.config = config
        self.args, self.kwargs = args, kwargs
        self.side_information = SimpleNamespace()
        tr = data_tuple[0]
        u_codes, users = pd.factorize(tr["userId"].to_numpy(), sort=False)            # first-appearance order
        order = np.argsort(u_codes, kind="stable")                                     # rows grouped by user, row order kept
        u_sorted = u_codes[order]
        it_sorted = tr["itemId"].to_numpy()[order]
        r_sorted = tr["rating"].to_numpy()[order]
        self.users = users.tolist()
        first_items = pd.unique(it_sorted)                                             # first occurrences, in dict-fill order
        seen = set()
        for x in first_items.tolist():                                                 # a real CPython set: its iteration
            seen.add(x)                                                                # order IS the reference's item order
        self.items = list(seen)
        self.num_users, self.num_items = len(self.users), len(self.items)
        self.private_users = dict(enumerate(self.users))
        self.public_users = {v: k for k, v in self.private_users.items()}
        self.private_items = dict(enumerate(self.items))
        self.public_items = {v: k for k, v in self.private_items.items()}
        i_sorted = pd.Index(self.items).get_indexer(it_sorted).astype(np.int64)
        u_sorted, i_sorted, r_sorted = self._dedup(u_sorted.astype(np.int64), i_sorted, r_sorted, self.num_items)
        self._tr = (u_sorted, i_sorted, r_sorted)                                      # private ids, dict order
        self.transactions = int(u_sorted.size)
        shape = (self.num_users, self.num_items)
        self.sp_i_train = sp.csr_matrix((np.ones(u_sorted.size, np.float32), (u_sorted, i_sorted)), dtype=np.float32, shape=shape)
        self.sp_i_train_ratings = sp.csr_matrix((r_sorted.astype(np.float32), (u_sorted, i_sorted)), dtype=np.float32, shape=shape)
        self._eval_frames = {"test": data_tuple[1] if len(data_tuple) == 2 else data_tuple[2]}
        if len(data_tuple) == 3:
            self._eval_frames["val"] = data_tuple[1]
        self._lazy = {}
        self._mask = None

    @staticmethod
    def _dedup(u, i, r, n_items):
        """(user, item) pairs once: first position, last rating (dict semantics).  Inputs are grouped by user."""
        key = u * np.int64(max(n_items, 1) + 1) + i
        uniq, first, inv = np.unique(key, return_index=True, return_inverse=True)
        if uniq.size == key.size:
            return u, i, r
        last_r = np.empty(uniq.size, dtype=r.dtype)
        last_r[inv] = r                                                                # later rows overwrite earlier ones
        keep = np.sort(first)
        return u[keep], i[keep], last_r[inv[keep]]

    # ---- dict views of the reference API, built on demand ---------------------------------
    def _dicts(self):
        if "train" not in self._lazy:
            u, i, r = self._tr
            users, items = self.users, self.items
            bounds = np.flatnonzero(np.diff(u, prepend=-1, append=self.num_users))     # group starts (+ end)
            pub, prv = {}, {}
            il, rl = i.tolist(), r.tolist()
            for g in range(len(bounds) - 1):
                a, b = int(bounds[g]), int(bounds[g + 1])
                pu = int(u[a])
                prv[pu] = dict(zip(il[a:b], rl[a:b]))
                pub[users[pu]] = {items[k]: v for k, v in prv[pu].items()}
            self._lazy["train"], self._lazy["i_train"] = pub, prv
        return self._lazy["train"], self._lazy["i_train"]

    @property
    def train_dict(self):
        return self._dicts()[0]

    @property
    def i_train_dict(self):
        return self._dicts()[1]

    def _split_dict(self, which):
        key = "dict_" + which
        if key not in self._lazy:
            df = self._eval_frames[which]
            raw = {}
            for u, i, r in zip(df["userId"].tolist(), df["itemId"].tolist(), df["rating"].tolist()):
                raw.setdefault(u, {})[i] = r
            self._lazy[key] = {u: raw.get(u, {}) for u in self.users}                  # every TRAIN user, dataset.py:257-262
        return self._lazy[key]

    @property
    def test_dict(self):
        return self._split_dict("test")

    def __getattr__(self, name):
        if name == "val_dict" and "val" in self.__dict__.get("_eval_frames", {}):
            return self._split_dict("val")
        raise AttributeError(name)

    def eval_arrays(self, which):
        """(private user, private item or -1, rating) of the split's rows whose user is a train user, grouped by user in
        train-user order, (user, item) duplicates reduced like a dict — the vectorised source of eval_csr_of."""
        if which not in self._eval_frames:
            return None
        df = self._eval_frames[which]
        pu = pd.Index(self.users).get_indexer(df["userId"].to_numpy())
        ok = pu >= 0
        pu = pu[ok].astype(np.int64)
        raw_items = df["itemId"].to_numpy()[ok]
        r = df["rating"].to_numpy()[ok]
        codes, _ = pd.factorize(raw_items, sort=False)                                 # dedup key must tell unknown items apart
        order = np.argsort(pu, kind="stable")
        pu, codes, raw_items, r = pu[order], codes[order].astype(np.int64), raw_items[order], r[order]
        key = pu * np.int64(codes.max(initial=0) + 2) + codes
        uniq, first, inv = np.unique(key, return_index=True, return_inverse=True)
        if uniq.size != key.size:
            last_r = np.empty(uniq.size, dtype=r.dtype); last_r[inv] = r
            keep = np.sort(first)
            pu, raw_items, r = pu[keep], raw_items[keep], last_r[inv[keep]]
        pi = pd.Index(self.items).get_indexer(raw_items).astype(np.int64)              # -1: test-only item
        return pu, pi, r

    # ---- reference accessors ---------------------------------------------------------------
    def get_test(self):
        return self.test_dict

    def get_validation(self):
        return getattr(self, "val_dict", None)

    @property
    def allunrated_mask(self):
        if self._mask is None:
            self._mask = np.where(self.sp_i_train.toarray() == 0, True, False)
        return self._mask

    # ---- kernel-side views (thin wrappers; the models call the free functions below, which also work on the
    # reference's own DataSet object when the plugin runs inside a real Elliot install) ----------------------
    def sampler_rows(self):
        return sampler_rows_of(self)

    def train_csr(self, device):
        return train_csr_of(self, device)

    def eval_csr(self, which="test"):
        return eval_csr_of(self, which)


# ---------------------------------------------------------------------------------------------------
# Kernel-side views of ANY object with the reference DataSet's fields (dataset.py:199-245): `i_train_dict`,
# `sp_i_train`, `users`, `public_items`, `test_dict` / `val_dict`, `config`.  They are free functions on purpose:
# inside a real Elliot install `self._data` is elliot.dataset.dataset.DataSet, which has none of the mirror's
# helper methods (ADVICE r1: the drop-in path must not depend on them).
# ---------------------------------------------------------------------------------------------------
def sampler_rows_of(data):
    """The reference sampler's `_ui_dict` (custom_sampler.py:21): per private user list(set(items)) — CPython set
    order, needed only where the reference's MT19937 stream is replayed (exact mode)."""
    if hasattr(data, "_tr"):                                          # the mirror: rows straight from the grouped arrays
        u, i, _ = data._tr
        bounds = np.flatnonzero(np.diff(u, prepend=-1, append=len(data.users)))
        il = i.tolist()
        rows = [[] for _ in range(len(data.users))]
        for g in range(len(bounds) - 1):
            a, b = int(bounds[g]), int(bounds[g + 1])
            # set(<dict>) pre-sizes its table from the dict's length, set(<list>) grows it insertion by insertion: the two
            # iterate in different orders, and the reference builds these from dicts (custom_sampler.py:21)
            rows[int(u[a])] = list(set(dict.fromkeys(il[a:b])))
        return rows
    return [list(set(data.i_train_dict[u])) for u in range(len(data.users))]


def train_csr_of(data, device, set_order=True):
    """(indptr int64, set-order indices int32 or None, sorted indices int32) on `device`, cached on the data object.
    The sorted CSR comes straight from `sp_i_train` (scipy, C speed — no per-row Python); the set-order copy is built
    row by row in Python because it IS CPython's set iteration order (exact mode only; set_order=False skips it)."""
    import torch
    cache = data.__dict__.setdefault("_eb200_dev", {})
    key = (str(device), bool(set_order))
    if key not in cache:
        other = cache.get((str(device), True))
        if other is not None:                                        # the full triple covers the partial request
            cache[key] = other
            return other
        m = data.sp_i_train.tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        indptr = m.indptr.astype(np.int64)
        srt = m.indices.astype(np.int32)
        flat = None
        if set_order:
            rows = sampler_rows_of(data)
            flat = np.fromiter((x for r in rows for x in r), dtype=np.int32, count=int(indptr[-1]))
            assert all(len(r) == indptr[u + 1] - indptr[u] for u, r in enumerate(rows)), "sp_i_train and i_train_dict disagree"
        cache[key] = tuple(None if a is None else torch.from_numpy(a).to(device) for a in (indptr, flat, srt))
    return cache[key]


def eval_csr_of(data, which="test"):
    """Host CSR (indptr, private item ids, gains) of the relevant items per private user (evaluator.py:117-147,
    relevance.py:80-82); None when the split does not exist."""
    thr = data.config.evaluation.relevance_threshold
    if hasattr(data, "eval_arrays"):                                  # the mirror: no dicts, no per-user Python
        arr = data.eval_arrays(which)
        if arr is None:
            return None
        pu, pi, r = arr
        keep = r >= thr
        pu, pi, r = pu[keep], pi[keep], r[keep]
        indptr = np.zeros(len(data.users) + 1, np.int64)
        np.cumsum(np.bincount(pu, minlength=len(data.users)), out=indptr[1:])
        return indptr, pi.astype(np.int64), (2.0 ** (r.astype(np.float64) - thr + 1) - 1).astype(np.float64)
    d = data.test_dict if which == "test" else getattr(data, "val_dict", None)
    if d is None:
        return None
    n_users = len(data.users)
    indptr = np.zeros(n_users + 1, np.int64)
    idx, gain = [], []
    for pu, u in enumerate(data.users):
        for it, score in d.get(u, {}).items():
            if score >= thr:
                idx.append(data.public_items.get(it, -1))            # test-only items can never be recommended
                gain.append(2 ** (score - thr + 1) - 1)              # relevance.py:80-82
        indptr[pu + 1] = len(idx)
    return indptr, np.array(idx, np.int64), np.array(gain, np.float64)


def eval_users_of(data, which="test"):
    """Boolean mask over private users: the user has any row in the split, whatever its rating (the users the reference
    Evaluator keeps, evaluator.py:117); None when the split does not exist."""
    if hasattr(data, "eval_arrays"):                                  # the mirror: no dicts
        arr = data.eval_arrays(which)
        if arr is None:
            return None
        return np.bincount(arr[0], minlength=len(data.users)) > 0
    d = data.test_dict if which == "test" else getattr(data, "val_dict", None)
    if d is None:
        return None
    return np.array([bool(d.get(u)) for u in data.users], dtype=bool)
