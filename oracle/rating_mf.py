"""fp64 NumPy restatements of the reference's SVD++ and FunkSVD train steps.  TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED, as oracle/tf_models.py: TensorFlow is absent, so these follow the reference's model code line by line
plus the TF 2.3 semantics it relies on.  What IS checked: the gradients against an fp64 torch autograd of the same
forward formulas (tests/test_oracle_rating.py), and the device step kernel against these (tests/test_gpu_rating_mf.py).
"""
import numpy as np


def implicit_means(P, Y, users, indptr, indices):
    """z_u = p_u + mean_{j in N(u)} y_j per listed user (svdpp_model.py:63: tf.map_fn of reduce_mean over the train row)."""
    return np.stack([P[u] + Y[indices[indptr[u]:indptr[u + 1]]].mean(0) for u in users]) if len(users) else P[:0]


def svdpp_forward_backward(T, u, i, y, indptr, indices, reg_w=0.1, reg_b=0.001):
    """SVDppModel.call/train_step (svdpp_model.py:58-82): out = (p_u + mean_{N(u)} y_j) . q_i + b_u + b_i + g, Keras
    MeanSquaredError (batch mean).  T: P, Q, Y (tables), bu, bi (vectors), g (scalar).  reg_w / reg_b are the Embedding
    regularizers the reference attaches and never adds to the differentiated loss: accepted, no effect.
    Returns loss, grads (same keys), out."""
    del reg_w, reg_b
    B = len(u)
    Z = implicit_means(T["P"], T["Y"], u, indptr, indices)
    out = (Z * T["Q"][i]).sum(1) + T["bu"][u] + T["bi"][i] + T["g"]
    loss = np.mean((out - y) ** 2)
    e = 2 * (out - y) / B
    G = {k: np.zeros_like(v) for k, v in T.items() if k != "g"}
    np.add.at(G["Q"], i, e[:, None] * Z)
    np.add.at(G["P"], u, e[:, None] * T["Q"][i])
    for s in range(B):
        row = indices[indptr[u[s]]:indptr[u[s] + 1]]
        np.add.at(G["Y"], row, e[s] * T["Q"][i[s]] / len(row))
    np.add.at(G["bu"], u, e)
    np.add.at(G["bi"], i, e)
    G["g"] = e.sum()
    return loss, G, out


def funk_svd_forward_backward(T, u, i, y, reg_w=0.1, reg_b=0.001):
    """FunkSVDModel.call/train_step (funk_svd_model.py:55-77): out = p_u . q_i + b_u + b_i, Keras MeanSquaredError.
    T: P, Q, bu, bi.  reg_w / reg_b: no effect, as for SVD++.  Returns loss, grads, out."""
    del reg_w, reg_b
    B = len(u)
    out = (T["P"][u] * T["Q"][i]).sum(1) + T["bu"][u] + T["bi"][i]
    loss = np.mean((out - y) ** 2)
    e = 2 * (out - y) / B
    G = {k: np.zeros_like(v) for k, v in T.items()}
    np.add.at(G["Q"], i, e[:, None] * T["P"][u])
    np.add.at(G["P"], u, e[:, None] * T["Q"][i])
    np.add.at(G["bu"], u, e)
    np.add.at(G["bi"], i, e)
    return loss, G, out


def rating_errors(lists, scores, rels, ratings):
    """The reference's MAE / MSE sums on explicit full lists (mae.py, mse.py): per user, over the list entries that are
    relevant items, |v - r| and (v - r)^2; the denominator counts every relevant item.  lists[u] / scores[u]: the full
    list and its scores, rels[u] / ratings[u]: relevant items (-1 test-only) and their test ratings."""
    a = q = 0.0
    n = 0
    for u in lists:
        r = dict(zip(rels[u], ratings[u]))
        n += len(rels[u])
        for it, v in zip(lists[u], scores[u]):
            if it in r:
                a += abs(v - r[it]); q += (v - r[it]) ** 2
    return a, q, n
