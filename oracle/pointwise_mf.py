"""fp64 NumPy restatements of the reference's MF, PMF, FM and LMF train steps, TF's Adagrad, the LMF epoch and each
model's full-list score.  TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED, as oracle/tf_models.py: TensorFlow is absent, so these follow the reference's model code line by line
plus the TF 2.3 semantics it relies on.  What IS checked: the gradients against an fp64 torch autograd of the same
forward formulas (tests/test_oracle_pointwise_mf.py), and the device kernels against these (tests/test_gpu_pointwise_mf.py).
"""
import numpy as np

ADAGRAD_INIT, ADAGRAD_EPS = 0.1, 1e-7


def sigmoid(x):
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def softplus(x):
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def mf_forward_backward(T, u, i, y):
    """MatrixFactorizationModel.train_step (matrix_factorization_model.py:52-71): out = p_u . q_i, Keras MeanSquaredError.
    T: P, Q.  The l2 Embedding regularizers never reach the differentiated loss.  Returns loss, grads, out."""
    B = len(u)
    out = (T["P"][u] * T["Q"][i]).sum(1)
    loss = np.mean((out - y) ** 2)
    e = 2 * (out - y) / B
    G = {k: np.zeros_like(v) for k, v in T.items()}
    np.add.at(G["Q"], i, e[:, None] * T["P"][u])
    np.add.at(G["P"], u, e[:, None] * T["Q"][i])
    return loss, G, out


def pmf_forward_backward(T, u, i, y):
    """ProbabilisticMatrixFactorizationModel.train_step (probabilistic_matrix_factorization_model.py:65-87) with the
    GaussianNoise layer inactive (called outside training mode): out = sigmoid(p_u . q_i), Keras MeanSquaredError."""
    B = len(u)
    o = sigmoid((T["P"][u] * T["Q"][i]).sum(1))
    loss = np.mean((o - y) ** 2)
    e = 2 * (o - y) * o * (1 - o) / B
    G = {k: np.zeros_like(v) for k, v in T.items()}
    np.add.at(G["Q"], i, e[:, None] * T["P"][u])
    np.add.at(G["P"], u, e[:, None] * T["Q"][i])
    return loss, G, o


def fm_forward_backward(T, u, i, y):
    """FactorizationMachineModel.train_step through MatrixFactorizationLayer (factorization_machine_model.py:62-72,
    285-291): out = p_u . q_i + g + b_u + b_i, Keras MeanSquaredError.  T: P, Q, bu, bi, g (scalar)."""
    B = len(u)
    out = (T["P"][u] * T["Q"][i]).sum(1) + T["g"] + T["bu"][u] + T["bi"][i]
    loss = np.mean((out - y) ** 2)
    e = 2 * (out - y) / B
    G = {k: np.zeros_like(v) for k, v in T.items() if k != "g"}
    np.add.at(G["Q"], i, e[:, None] * T["P"][u])
    np.add.at(G["P"], u, e[:, None] * T["Q"][i])
    np.add.at(G["bu"], u, e)
    np.add.at(G["bi"], i, e)
    G["g"] = e.sum()
    return loss, G, out


def lmf_forward_backward(T, u, i, y, alpha, reg):
    """LogisticMatrixFactorizationModel.train_step (logistic_matrix_factorization_model.py:65-90), item branch:
    x = g_u . g_i + b_u + b_i; loss = sum -(alpha y x - (1 + alpha y) log(1 + e^x)) + reg (l2_loss(g_u) + l2_loss(g_i))
    over the looked-up rows (softplus in a stable form); gradients of Gi and Bi only.  T: Gu, Gi, Bu, Bi."""
    x = (T["Gu"][u] * T["Gi"][i]).sum(1) + T["Bu"][u] + T["Bi"][i]
    ay = alpha * y
    loss = np.sum(-(ay * x - (1 + ay) * softplus(x))) + reg * (0.5 * (T["Gu"][u] ** 2).sum() + 0.5 * (T["Gi"][i] ** 2).sum())
    c = sigmoid(x) * (1 + ay) - ay
    G = {"Gi": np.zeros_like(T["Gi"]), "Bi": np.zeros_like(T["Bi"])}
    np.add.at(G["Gi"], i, c[:, None] * T["Gu"][u] + reg * T["Gi"][i])
    np.add.at(G["Bi"], i, c)
    return loss, G, x


def adagrad_dense(var, acc, grad, lr, eps=ADAGRAD_EPS):
    """ResourceApplyAdagradV2: acc += g^2; var -= lr g / (sqrt(acc) + eps), every element (in place)."""
    acc += grad * grad
    var -= lr * grad / (np.sqrt(acc) + eps)


def adagrad_sparse(var, acc, rows, row_grads, lr, eps=ADAGRAD_EPS):
    """Keras Adagrad on IndexedSlices: duplicate indices summed (_deduplicate_indexed_slices), then
    ResourceSparseApplyAdagradV2 on each distinct row once (in place)."""
    uniq, inv = np.unique(rows, return_inverse=True)
    g = np.zeros((len(uniq),) + var.shape[1:])
    np.add.at(g, inv, row_grads)
    acc[uniq] += g * g
    var[uniq] -= lr * g / (np.sqrt(acc[uniq]) + eps)


def lmf_epoch(T, acc, stream, T_samples, batch, alpha, reg, lr):
    """One LMF epoch (logistic_matrix_factorization.py:92-112): two passes of T_samples samples, both item steps, taken
    from `stream` (u, i, y arrays of at least 2 T_samples, continuing from the first pass to the second); Adagrad on Gi,
    Bi in place; returns the summed loss."""
    u, i, y = stream
    total = 0.0
    for p in range(2):
        for s in range(p * T_samples, (p + 1) * T_samples, batch):
            e = min(s + batch, (p + 1) * T_samples)
            loss, G, _ = lmf_forward_backward(T, u[s:e], i[s:e], y[s:e], alpha, reg)
            total += loss
            for k in ("Gi", "Bi"):
                adagrad_dense(T[k], acc[k], G[k], lr)
    return total


def rating_labels(indptr, indices, ratings, u, i, y):
    """pointwise_pos_neg_ratings_sampler.py's labels on the pointwise sampler's draws: a positive (y != 0) carries the
    train rating of (u, i), a negative keeps 0."""
    out = np.array(y, dtype=np.float64)
    for s in range(len(u)):
        if out[s] != 0:
            row = indices[indptr[u[s]]:indptr[u[s] + 1]]
            p = np.searchsorted(row, i[s])
            assert p < len(row) and row[p] == i[s], "a positive must be in the train row"
            out[s] = ratings[indptr[u[s]] + p]
    return out


def full_scores(model, T):
    """[n_users][n_items] fp64 full-list scores: MF p.q, PMF sigmoid(p.q), FM p.q + b_u + b_i + g, LMF b_u + b_i + g_u.g_i
    (get_recs / predict_batch)."""
    if model == "LMF":
        return T["Bu"][:, None] + T["Bi"][None, :] + T["Gu"] @ T["Gi"].T
    s = T["P"] @ T["Q"].T
    if model == "PMF":
        return sigmoid(s)
    if model == "FM":
        return s + T["bu"][:, None] + T["bi"][None, :] + T["g"]
    return s
