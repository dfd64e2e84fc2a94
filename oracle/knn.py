"""fp64 restatement of the reference's ItemKNN / UserKNN, standard implementation (item_knn_similarity.py:34-78,
user_knn_similarity.py:33-77, get_user_recs :157-174), with the tie rules of the device kernels:

  gram        G = R^T R (items) or R R^T (users), exact in fp64 for the ratings the device path accepts;
  similarity  cosine = fp32(G_rc / sqrt(G_rr * G_cc)) (0 when a norm is 0), dot = fp32(G_rc);
  neighbours  per row the k largest NONZERO values, value desc then column asc (the row itself included);
  preds       R . W (items) or W . R (users) in fp64, W[x, y] = value of x in y's list;
  topk        train items -> -inf, the k best by (score desc, column asc), -1 padded when fewer are unmasked.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import numpy as np


def gram(R, over):
    R = np.asarray(R, dtype=np.float64)
    return R.T @ R if over == "items" else R @ R.T


def similarity(G, cosine):
    if not cosine:
        return G.astype(np.float32)
    d = np.diag(G).astype(np.float64)
    den = np.sqrt(np.outer(d, d))
    with np.errstate(divide="ignore", invalid="ignore"):
        S = np.where(den > 0, G / np.where(den > 0, den, 1.0), 0.0)
    return S.astype(np.float32)


def neighbours(S, k):
    """(idx int32 [n][k], val fp32 [n][k], cnt [n]) of every row of S."""
    n = S.shape[0]
    idx = np.full((n, k), -1, np.int32)
    val = np.zeros((n, k), np.float32)
    cnt = np.zeros(n, np.int32)
    cols = np.arange(S.shape[1])
    for r in range(n):
        v = S[r]
        nz = np.flatnonzero(v != 0)
        order = nz[np.lexsort((cols[nz], -v[nz].astype(np.float64)))][:k]
        m = len(order)
        idx[r, :m], val[r, :m], cnt[r] = order, v[order], m
    return idx, val, cnt


def weights(idx, val):
    n = idx.shape[0]
    W = np.zeros((n, n), np.float64)
    ok = idx >= 0
    y = np.repeat(np.arange(n), idx.shape[1]).reshape(idx.shape)
    W[idx[ok], y[ok]] = val[ok]
    return W


def preds(R, idx, val, over):
    R = np.asarray(R, dtype=np.float64)
    W = weights(idx, val)
    return R @ W if over == "items" else W @ R


def topk(P, train_mask, k):
    """train_mask: bool [users][items], True = train item."""
    P = np.where(train_mask, -np.inf, P)
    n, m = P.shape
    idx = np.full((n, k), -1, np.int64)
    val = np.full((n, k), -np.inf)
    cols = np.arange(m)
    for u in range(n):
        ok = np.flatnonzero(~train_mask[u])
        order = ok[np.lexsort((cols[ok], -P[u, ok]))][:k]
        idx[u, :len(order)], val[u, :len(order)] = order, P[u, order]
    return idx, val


def isolated(v, v_next, rel=1e-5):
    """Ranks whose value is more than 2 * rel (relative) away from both neighbours; v_next: the (k+1)-th values."""
    w = np.concatenate([v, v_next[:, None]], 1)
    t = rel * np.maximum(np.abs(w), 1e-30)
    with np.errstate(invalid="ignore"):
        gap = np.abs(w[:, :-1] - w[:, 1:])
        ok = gap > 2 * t[:, :-1]
    iso = np.isfinite(v) & ok
    iso[:, 1:] &= ok[:, :-1]
    return iso


def run(R, over, k_nn, cosine, k):
    """Everything for a dense rating matrix R [users][items]: (neighbour idx, val, cnt, preds, top-k idx, top-k val)."""
    S = similarity(gram(R, over), cosine)
    idx, val, cnt = neighbours(S, k_nn)
    P = preds(R, idx, val, over)
    ti, tv = topk(P, np.asarray(R) != 0, k)
    return idx, val, cnt, P, ti, tv
