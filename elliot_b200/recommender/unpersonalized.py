"""MostPop and Random, the reference's unpersonalized baselines (recommender/unpersonalized/most_popular/most_popular.py,
random_recommender/Random.py; external/models/most_popular behaves as most_popular.py), on the H100.

MostPop: pop[i] = train users of item i, one global order (pop desc, item asc: Python's stable sort of the reference),
and per user the first k items of that order that are not train items, scored with pop as a Python int.  A user with
|train_u| + k >= n_items gets no list: the reference stores `r[u] = []` under the user's PRIVATE id and leaves its
public id out, so a real user whose public id equals that private id ends up with [] when its own private id is smaller
(the later write wins) and keeps its list otherwise.  The dict path rebuilds exactly that dict; device evaluation
(`b200_eval: device`) falls back to it for an evaluation where the quirk fires, so that absent users stay absent.

Random (`random_seed`, default 42; name Random_seed=<seed>): np.random.seed(random_seed) in the constructor, then per
user in private order min(k, n_u) draws r = np.random.randint(n_u) with replacement (n_u = items outside the train row),
each listing the r-th such item in ascending private order with the int score 1.  The draws replay numpy's legacy
MT19937 stream on the device (ops.RandomStream), which persists, so a second evaluation continues the stream.

Both models have no `_model`: with meta.save_weights the reference's RecMixin logs "Saving weights FAILED", and so does
this build.  AUC / GAUC are refused in the constructor (init_charger), and evaluation-time negative sampling raises
NotImplementedError.
"""
import time

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import cuda_device


class MostPopLists:
    """The popularity, the global order and the MostPop lists on the device."""

    def __init__(self, data, device="cuda:0"):
        self.device = torch.device(device)
        self.n_items = len(data.items)
        self.indptr, _, self.train = train_csr_of(data, self.device, set_order=False)
        self.n_train = np.diff(data.sp_i_train.tocsr().indptr)
        self.pop = self.order = None

    def initialize(self, mark=None):
        """pop and order.  `mark(phase)`, when given, is called as each phase's work has been queued (popularity,
        order), so that a caller can time the phases with CUDA events."""
        mark = mark or (lambda phase: None)
        self.pop = ops.item_pop(self.train, self.n_items)
        mark("popularity")
        self.order = torch.sort(self.pop, descending=True, stable=True).indices.to(torch.int32)
        mark("order")

    def skips(self, k):
        """True when some user has |train_u| + k >= n_items (the reference lists nothing for it)."""
        return bool(self.n_train.size) and int(self.n_train.max()) + k >= self.n_items

    def topk(self, k, users=None, mark=None):
        """(idx int32, pop int32) [rows][k]; rows of skipped users are -1."""
        idx, val, _ = ops.mostpop_topk(self.order, self.pop, k, self.indptr, self.train, users=users)
        if mark:
            mark("lists")
        return idx, val


class RandomLists:
    """The device stream of np.random.seed(seed) and the Random lists drawn from it."""

    def __init__(self, data, seed, device="cuda:0"):
        self.device = torch.device(device)
        self.n_items = len(data.items)
        self.indptr, _, self.train = train_csr_of(data, self.device, set_order=False)
        self.stream = ops.RandomStream(seed, self.device)

    def topk(self, k, users=None, mark=None):
        """(idx int32, score int32 = 1) [rows][k], -1 / 0 past min(k, n_u).  Every call draws for every user, in
        order, whatever `users` selects: that is where the reference's stream goes."""
        mark = mark or (lambda phase: None)
        r = self.stream.draws(k, self.indptr, self.n_items)
        mark("stream")
        idx = ops.complement_select(r, self.indptr, self.train, users=users)
        mark("select")
        return idx, (idx >= 0).to(torch.int32)


def int_lists(data, idx, val, first=0):
    """Per row r (private user first + r): the reference's [(public item, int score), ...], -1 slots skipped."""
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    items = np.array(data.items, dtype=object)
    return [list(zip(items[i[i >= 0]].tolist(), v[i >= 0].tolist())) for i, v in zip(idx, val)]


class _ListRecs:
    """The recommendation methods of both models; `_lists.topk(k)` gives every user's row."""

    def get_recommendations(self, k: int = 10):
        recs_val, recs_test = self.process_protocol(k)
        return dict(recs_val), dict(recs_test)

    def get_recommendations_tensors(self, k: int = 10):
        """(idx, score) device tensors, rows = private users, -1 padded."""
        return self._lists.topk(k)

    def get_single_recommendation(self, mask, k, *args):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        return self._dict(k, int_lists(self._data, *self.get_recommendations_tensors(k)))


class MostPop(_ListRecs, RecMixin, BaseRecommenderModel):
    r"""Most popular items, on the H100.  YAML block as the reference's: MostPop: {meta: {...}}; optional keys
    `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._device = cuda_device(self._params, "MostPop")
        self._lists = MostPopLists(self._data, self._device)

    @property
    def name(self):
        return "MostPop"

    def train(self):
        start = time.time()
        self._lists.initialize()
        torch.cuda.synchronize(self._device)
        self.logger.info(f"The popularity order has taken: {time.time() - start}")
        self.evaluate()

    def lists_are_tensors(self, k):
        """False when the reference leaves some user out of its lists at cutoff k: evaluation then takes the dict."""
        return not self._lists.skips(k)

    def _dict(self, k, lists):
        # most_popular.py: users in private order; a user the reference skips is written as [] under its PRIVATE id
        n_train, n_items = self._lists.n_train, self._lists.n_items
        r = {}
        for u, (pub, lst) in enumerate(zip(self._data.users, lists)):
            if n_train[u] + k >= n_items:
                r[u] = []
            else:
                r[pub] = lst
        return r


class Random(_ListRecs, RecMixin, BaseRecommenderModel):
    r"""Random items, on the H100.  YAML block as the reference's: Random: {meta: {...}, random_seed: 42}; optional
    keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [("_seed", "random_seed", "seed", 42, int, None)]
        self.autoset_params()
        np.random.seed(self._seed)
        self._device = cuda_device(self._params, "Random")
        self._lists = RandomLists(self._data, self._seed, self._device)

    @property
    def name(self):
        return f"Random_{self.get_params_shortcut()}"

    def train(self):
        self.evaluate()

    def _dict(self, k, lists):
        return dict(zip(self._data.users, lists))
