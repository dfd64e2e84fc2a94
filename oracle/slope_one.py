"""fp64 restatement of the reference's SlopeOne (algebric/slope_one/slope_one_model.py:19-64), with the tie rule of the
device kernels:

  counts      F[i, j] = number of users with entries for both i and j (an explicit 0 rating is an entry);
  deviations  D[i, j] = sum_u (r_ui - r_uj) = (X^T B - B^T X)[i, j], with X the ratings and B the entry pattern: exact
              fp64 products of dyadic ratings, so any summation order gives the same D;
              E[i, j] = D[i, j] / F[i, j] rounded once, NaN where F = 0;
              the reference's `dev` is E above the diagonal, -E^T below it, 0 on the diagonal and where F = 0;
  means       np.mean of each user's ratings, as the reference takes it;
  scores      pred[u, c] = mean_u + (sum_j -E[j, c]) / n over the user's train items j in the given (dict) order, NaN
              terms skipped and n counting the rest; mean_u when n = 0.  The sum is plain sequential fp64 addition,
              vectorised over the candidates c one train item at a time;
  topk        train items excluded, the k best by (score desc, item asc), -1 / -inf padded.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import zlib

import numpy as np


def dense(indptr, items, ratings, n_items):
    """(X ratings fp64, B entry pattern fp64) [n_users][n_items] of a CSR whose rows may be in any order."""
    n_users = len(indptr) - 1
    X = np.zeros((n_users, n_items))
    B = np.zeros((n_users, n_items))
    rows = np.repeat(np.arange(n_users), np.diff(indptr))
    X[rows, items] = ratings
    B[rows, items] = 1.0
    return X, B


def deviations(indptr, items, ratings, n_items):
    """(F, E): the co-rating counts and the deviations D / F (NaN where F = 0), both fp64 [n_items][n_items]."""
    X, B = dense(indptr, items, ratings, n_items)
    F = B.T @ B
    D = X.T @ B - B.T @ X
    with np.errstate(divide="ignore", invalid="ignore"):
        E = np.where(F > 0, D / np.where(F > 0, F, 1.0), np.nan)
    return F, E


def reference_dev(E):
    """The reference's `dev` array from E: upper triangle E, lower triangle its negation, 0 on the diagonal and where no
    user rated both items."""
    n = E.shape[0]
    dev = np.triu(np.nan_to_num(E, nan=0.0), 1)
    iu = np.triu_indices(n, 1)
    dev[iu[1], iu[0]] = -dev[iu]                    # the reference negates the upper value (0 -> -0.0)
    return dev


def sorted_rows(indptr, items, ratings):
    """(items, ratings) with every row's entries sorted by item: the summation order the reference does NOT use."""
    items, ratings = items.copy(), ratings.copy()
    for u in range(len(indptr) - 1):
        a, b = indptr[u], indptr[u + 1]
        o = np.argsort(items[a:b], kind="stable")
        items[a:b], ratings[a:b] = items[a:b][o], ratings[a:b][o]
    return items, ratings


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a, dtype=np.float64).tobytes())


def user_means(indptr, ratings):
    return np.array([np.mean([float(r) for r in ratings[indptr[u]:indptr[u + 1]]])
                     for u in range(len(indptr) - 1)], dtype=np.float64)


def scores(E, means, indptr, items, users=None):
    """pred[q, c] for the users `users` (default all), every column c of E, summed in the CSR's stored order (the
    items index the rows of E)."""
    users = np.arange(len(indptr) - 1) if users is None else np.asarray(users)
    out = np.empty((len(users), E.shape[1]))
    for q, u in enumerate(users):
        s = np.zeros(E.shape[1])
        n = np.zeros(E.shape[1], np.int64)
        for j in items[indptr[u]:indptr[u + 1]]:
            e = E[j]
            ok = ~np.isnan(e)
            s = np.where(ok, s + (-np.where(ok, e, 0.0)), s)
            n += ok
        with np.errstate(divide="ignore", invalid="ignore"):
            out[q] = np.where(n > 0, means[u] + s / np.maximum(n, 1), means[u])
    return out


def topk(P, indptr, items, k, users=None):
    """(idx [n][k] int64, val [n][k] fp64): each row's train items excluded, (score desc, item asc), -1 / -inf padded."""
    users = np.arange(len(indptr) - 1) if users is None else np.asarray(users)
    idx = np.full((len(users), k), -1, np.int64)
    val = np.full((len(users), k), -np.inf)
    for q, u in enumerate(users):
        cand = np.setdiff1d(np.arange(P.shape[1]), items[indptr[u]:indptr[u + 1]])
        order = np.lexsort((cand, -P[q, cand]))[:k]
        idx[q, :len(order)] = cand[order]
        val[q, :len(order)] = P[q, cand[order]]
    return idx, val


def isolated(val, margin=0.0):
    """Ranks whose value differs (by more than `margin`) from both neighbours' in the row: there the list position of
    an item does not depend on the tie rule."""
    v = np.asarray(val, dtype=np.float64)
    pad = np.full((v.shape[0], 1), np.nan)
    prev = np.concatenate([pad, v[:, :-1]], 1)
    nxt = np.concatenate([v[:, 1:], pad], 1)
    with np.errstate(invalid="ignore"):
        far = lambda a, b: ~(np.abs(a - b) <= margin)   # a NaN neighbour (row end, -inf padding) counts as far
        return far(v, prev) & far(v, nxt) & np.isfinite(v)
