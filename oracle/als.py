"""fp64 numpy restatement of the reference's iALS and WRMF (latent_factor_models/iALS/iALS_model.py,
latent_factor_models/WRMF/wrmf_model.py), written from their formulas, for the goldens of tests/golden/als_*.npz:

  confidences: float32 as the reference computes them on its float32 `sp_i_train`;
  iALS step:   G = Y^T Y, every user solved; G = X^T X of the NEW X, only items with train entries solved;
  WRMF step:   G_y = Y^T Y and G_x = X^T X both before the user half, every user then every item solved
               (an item without entries gets b = 0, so y = 0);
  per row:     x_r = (G + sum_e w_e y_e y_e^T + reg I)^-1 sum_e c_e y_e, by an explicit inverse (iALS) or an LU
               solve (WRMF) as the reference does;
  top k:       X Y^T, train items masked, (score desc, item asc).
"""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.linalg import spsolve


def ials_confidences(data, alpha, epsilon, scaling):
    C = np.array(data, dtype=np.float32)
    if scaling == "linear":
        C = np.float32(1.0) + np.float32(alpha) * C
    elif scaling == "log":
        C = np.float32(1.0) + np.float32(alpha) * np.log(np.float32(1.0) + C / np.float32(epsilon))
    return (C - np.float32(1)).astype(np.float64), C.astype(np.float64)


def wrmf_confidences(data, alpha):
    C = np.float32(alpha) * np.array(data, dtype=np.float32)
    w = C.astype(np.float64)
    return w, np.where(C != 0, w + 1.0, 0.0)


def _half(G, other, indptr, indices, w, c, reg, rows, out, solve):
    d = G.shape[0]
    for r in rows:
        s = slice(indptr[r], indptr[r + 1])
        P = other[indices[s]]
        A = G + (P * w[s][:, None]).T @ P + reg * np.eye(d)
        out[r] = solve(A, P.T @ c[s])


def _inv_dot(A, b):                 # iALS_model.py:54: np.dot(np.linalg.inv(B), b)
    return np.linalg.inv(A) @ b


def _lu(A, b):                      # wrmf_model.py:50: spsolve, an LU factorisation
    return spsolve(sp.csc_matrix(A), b)


def train(kind, R, X0, Y0, epochs, alpha, reg, epsilon=1.0, scaling="linear"):
    """R: csr train matrix (float32 values); returns [(X, Y) after each epoch] and the confidences (w, c) in R's order."""
    R = sp.csr_matrix(R, dtype=np.float32)
    R.sort_indices()
    w, c = ials_confidences(R.data, alpha, epsilon, scaling) if kind == "iALS" else wrmf_confidences(R.data, alpha)
    T = sp.csr_matrix((np.arange(R.nnz), R.indices, R.indptr), shape=R.shape).tocsc()
    perm = T.data
    X, Y = X0.astype(np.float64).copy(), Y0.astype(np.float64).copy()
    users = range(R.shape[0])
    items = [i for i in range(R.shape[1]) if T.indptr[i + 1] > T.indptr[i]] if kind == "iALS" else range(R.shape[1])
    solve = _inv_dot if kind == "iALS" else _lu
    out = []
    for _ in range(epochs):
        Gy = Y.T @ Y
        Gx_stale = X.T @ X
        _half(Gy, Y, R.indptr, R.indices, w, c, reg, users, X, solve)
        Gx = X.T @ X if kind == "iALS" else Gx_stale
        _half(Gx, X, T.indptr, T.indices, w[perm], c[perm], reg, items, Y, solve)
        out.append((X.copy(), Y.copy()))
    return out, (w, c)


def topk(X, Y, train_mask, k):
    S = X @ Y.T
    S[train_mask] = -np.inf
    idx = np.lexsort((np.broadcast_to(np.arange(S.shape[1]), S.shape), -S), axis=1)[:, :k]
    return idx, np.take_along_axis(S, idx, 1)
