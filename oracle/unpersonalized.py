"""NumPy restatement of the reference's MostPop and Random lists (recommender/unpersonalized/), on private ids.

Both take the train CSR (indptr, indices; any order within a row) of the private users and n_items, and return rows
of private item ids, -1 past the end of a list.
"""
import numpy as np


def popularity(indptr, indices, n_items):
    """pop[i] = train users of item i, and the order (pop desc, item asc) the reference's stable sort gives."""
    pop = np.bincount(np.asarray(indices, np.int64), minlength=n_items).astype(np.int64)
    return pop, np.argsort(-pop, kind="stable")


def mostpop(indptr, indices, n_items, k):
    """(rows [n_users][k], scores = pop, skipped [n_users] bool): the first k items of the order outside each train
    row; a user with |train_u| + k >= n_items is skipped (an empty row)."""
    pop, order = popularity(indptr, indices, n_items)
    n_users = len(indptr) - 1
    rows = np.full((n_users, k), -1, np.int64)
    skipped = np.diff(indptr) + k >= n_items
    for u in np.flatnonzero(~skipped):
        cand = order[~np.isin(order, indices[indptr[u]:indptr[u + 1]])][:k]
        rows[u, :len(cand)] = cand
    return rows, np.where(rows >= 0, pop[np.maximum(rows, 0)], 0), skipped


class Stream:
    """numpy's legacy MT19937 stream of np.random.seed(seed) as raw 32-bit words, and randint(n) read from it by the
    masked rejection of the legacy generator (randint(1) reads nothing)."""

    def __init__(self, seed, chunk=1 << 16):
        self._rs = np.random.RandomState(seed)
        self._chunk, self._buf, self._at, self.consumed = chunk, np.empty(0, np.uint32), 0, 0

    def _word(self):
        if self._at == len(self._buf):
            self._buf, self._at = self._rs.randint(0, 2 ** 32, size=self._chunk, dtype=np.uint32), 0
        self._at += 1
        self.consumed += 1
        return int(self._buf[self._at - 1])

    def randint(self, n):
        rng = n - 1
        if rng == 0:
            return 0
        mask = (1 << int(rng).bit_length()) - 1
        while True:
            v = self._word() & mask
            if v <= rng:
                return v


def random_draws(stream, indptr, n_items, k):
    """r [n_users][k]: each user's min(k, n_u) draws randint(n_u), in user order, -1 after them."""
    n_users = len(indptr) - 1
    r = np.full((n_users, k), -1, np.int64)
    for u in range(n_users):
        n_u = n_items - int(indptr[u + 1] - indptr[u])
        for j in range(min(k, n_u)):
            r[u, j] = stream.randint(n_u)
    return r


def complement_select(r, indptr, indices, n_items):
    """The r-th item outside each user's train row, -1 where r < 0."""
    out = np.full(r.shape, -1, np.int64)
    for u in range(r.shape[0]):
        free = np.setdiff1d(np.arange(n_items), indices[indptr[u]:indptr[u + 1]])
        ok = r[u] >= 0
        out[u, ok] = free[r[u, ok]]
    return out
