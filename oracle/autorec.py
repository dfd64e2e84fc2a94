"""fp64 restatements of UserAutoRec / ItemAutoRec (neural/UserAutoRec/userautorec_model.py, neural/ItemAutoRec/
itemautorec_model.py, itemautorec.py:99-108) and a replay of the models' Python `random` call sequence.

Weights are in Keras's layouts here: W1 [n_in][H], W2 [H][n_out] (recommender/autorec.py stores W2 transposed).
act is "linear" (UserAutoRec's decoder) or "sigmoid" (ItemAutoRec's).
"""
import random

import numpy as np


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _act(o, act):
    return sigmoid(o) if act == "sigmoid" else o


def init_biases(H, n_out):
    """Both Dense layers' biases: keras.initializers.Ones()."""
    return np.ones(H), np.ones(n_out)


def forward(X, W1, b1, W2, b2, act):
    """(h, o, reconstruction) of call() on dense input rows X [B][n_in]."""
    h = sigmoid(X @ W1 + b1)
    o = h @ W2 + b2
    return h, o, _act(o, act)


def step(X, W1, b1, W2, b2, act, h=None):
    """train_step (userautorec_model.py:93-107) on the dense batch X, literally: reconstructed * sign(X), error, the
    row sums of its squares and their mean.  Returns (loss, dW1, db1, dW2, db2).  h: the encoder output to run the
    decoder on (default: sigmoid(X W1 + b1))."""
    B = X.shape[0]
    if h is None:
        h = sigmoid(X @ W1 + b1)
    o = h @ W2 + b2
    rec = _act(o, act)
    s = np.sign(X)
    err = X - rec * s
    loss = (err ** 2).sum(1).mean()
    drec = -2.0 * err * s / B
    do = drec * (rec * (1.0 - rec) if act == "sigmoid" else 1.0)
    dW2, db2 = h.T @ do, do.sum(0)
    dpre1 = (do @ W2.T) * h * (1.0 - h)
    return loss, X.T @ dpre1, dpre1.sum(0), dW2, db2


def top_k(scores, mask, k):
    """tf.nn.top_k(tf.where(mask, scores, -inf), k): (values, ids) per row, the lower index first among equal values."""
    s = np.where(mask, scores, -np.inf)
    ids = np.argsort(-s, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(s, ids, 1), ids


def get_recommendations_user(X, W1, b1, W2, b2, mask, k, block):
    """RecMixin.get_recommendations (recommender_utils_mixin.py:63-73): predict on the dense train rows in user blocks,
    then the masked top_k (mask = allunrated_mask: True where an item may be listed)."""
    vals, ids = [], []
    for o in range(0, X.shape[0], block):
        e = min(o + block, X.shape[0])
        v, i = top_k(forward(X[o:e], W1, b1, W2, b2, "linear")[2], mask[o:e], k)
        vals.append(v); ids.append(i)
    return np.concatenate(vals), np.concatenate(ids)


def get_recommendations_item(XT, W1, b1, W2, b2, perm, mask, k):
    """ItemAutoRec.get_recommendations (itemautorec.py:99-108): the item rows XT[perm] reconstructed, the I x U
    predictions transposed, column j taken as item j, masked and top_k."""
    pred = forward(XT[np.asarray(perm)], W1, b1, W2, b2, "sigmoid")[2]
    return top_k(pred.T, mask, k)


def user_scores(X, W1, b1, W2, b2):
    """The factorised UserAutoRec scores: (h [U][H], W2^T [I][H], b2), score = h W2 + b2."""
    h = sigmoid(X @ W1 + b1)
    return h, W2.T, b2


def item_operands(XT, W1, b1, W2, b2, perm):
    """The factorised ItemAutoRec scores: (W2^T [U][H], V [I][H] with V[j] = g_perm[j], b2 [U]); score of (u, j) =
    sigmoid(W2^T[u] . V[j] + b2[u])."""
    V = sigmoid(XT[np.asarray(perm)] @ W1 + b1)
    return W2.T, V, b2


def replay(n_rows, n_items, epochs, item, validation_rate=1):
    """The models' draws on the `random` stream after `random.seed(42)` at construction: one random.sample(range(n_rows),
    n_rows) per epoch (sparse_sampler.py:18), and for ItemAutoRec one random.sample(range(n_items), n_items) per
    evaluation (itemautorec.py:102).  Returns [(kind, epoch, permutation)] in stream order; the global stream is restored."""
    state = random.getstate()
    try:
        random.seed(42)
        out = []
        for e in range(epochs):
            out.append(("epoch", e, random.sample(range(n_rows), n_rows)))
            if item and (e + 1) % validation_rate == 0:
                out.append(("eval", e, random.sample(range(n_items), n_items)))
        return out
    finally:
        random.setstate(state)


def replay_restore(n_items):
    """The permutation a restored ItemAutoRec evaluates under: the first draw after construction."""
    state = random.getstate()
    try:
        random.seed(42)
        return random.sample(range(n_items), n_items)
    finally:
        random.setstate(state)
