"""fp64 restatement of the reference's EASE^R (autoencoders/EASE_R/ease_r.py:69-95, get_user_predictions :52-67), with the
tie rule of the device kernels:

  gram     G = R^T R in fp64 (exact for the ratings the device path accepts);
  diag     G[j, j] = fp32(count_j + l2_norm), count_j = number of train ratings of item j (ease_r.py:85-87: the int64
           popularity plus the Python float, stored into the float32 matrix);
  inverse  P = G^-1 in fp64;
  weights  B[i, j] = fp32(-P[i, j] / P[j, j]), B[j, j] = 0 (ease_r.py:89-91, rounded to the reference's float32 once);
  preds    R . B in fp64 over the fp32 B;
  topk     train items -> -inf, the k best by (score desc, column asc), -1 padded (oracle/knn.py).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import numpy as np

from oracle.knn import topk  # noqa: F401  (re-exported: the same masked top-k)


def normal_matrix(R, l2_norm):
    R = np.asarray(R, dtype=np.float64)
    G = R.T @ R
    count = (R != 0).sum(0)
    G[np.diag_indices(G.shape[0])] = (count + float(l2_norm)).astype(np.float32)
    return G


def weights(P):
    d = np.diag(P).copy()
    B = (-P / d[None, :]).astype(np.float32)
    B[np.diag_indices(B.shape[0])] = 0.0
    return B


def preds(R, B):
    return np.asarray(R, dtype=np.float64) @ B.astype(np.float64)


def run(R, l2_norm, k):
    """Everything for a dense rating matrix R [users][items]: (fp32 B, preds, top-k idx, top-k val)."""
    B = weights(np.linalg.inv(normal_matrix(R, l2_norm)))
    P = preds(R, B)
    ti, tv = topk(P, np.asarray(R) != 0, k)
    return B, P, ti, tv
