"""fp64 restatements of DMF (neural/DMF/deep_matrix_factorization_model.py) and a host restatement of its sampler
(dataset/samplers/pointwise_pos_neg_ratio_ratings_sampler.py).

Tower weights follow recommender/dmf.py: W[0] is [n_in][w0] (the first layer's Keras kernel), W[l] for l >= 1 is
[w_l][w_(l-1)] (the transposed Keras kernel), b[l] has w_l entries (longer arrays are cut).
"""
import numpy as np

L2_EPS = 1e-12
# Keras's BinaryCrossentropy runs in float32: epsilon() becomes float32(1e-7), and the clip's upper bound
# float32(1) - float32(1e-7) = 1 - 2^-23 + ..., not 1 - 1e-7
BCE_EPS = float(np.float32(1e-7))
BCE_HI = float(np.float32(1) - np.float32(1e-7))


def tower(X, W, b):
    """Forward of one tower on dense input rows X [B][n_in]: (output, [pre-activations], [activations])."""
    pres, acts = [], []
    h = X
    for l, w in enumerate(W):
        z = h @ (w if l == 0 else w.T) + b[l][:w.shape[1] if l == 0 else w.shape[0]]
        pres.append(z)
        h = np.maximum(z, 0.0) if l < len(W) - 1 else z
        acts.append(h)
    return h, pres, acts


def tower_backward(X, W, pres, acts, d):
    """Gradients (dW, db) of one tower from d = dloss/doutput."""
    dW, db = [None] * len(W), [None] * len(W)
    for l in range(len(W) - 1, -1, -1):
        if l < len(W) - 1:
            d = d * (pres[l] > 0)
        inp = X if l == 0 else acts[l - 1]
        dW[l] = inp.T @ d if l == 0 else d.T @ inp
        db[l] = d.sum(0)
        if l > 0:
            d = d @ W[l]
    return dW, db


def l2_normalize_cols(x):
    """tf.nn.l2_normalize(x, 0): (x / sqrt(max(sum_b x^2, 1e-12)), inverse norms, mask of the columns above the floor)."""
    ss = (x * x).sum(0)
    inv = 1.0 / np.sqrt(np.maximum(ss, L2_EPS))
    return x * inv, inv, ss >= L2_EPS


def head(U, V, label, max_rating, cosine):
    """(mean loss, dU, dV, outputs) of the clipped BCE on sum_f u^ v^ (Keras BinaryCrossentropy, batch mean; clip_by_value
    passes the gradient on the closed interval)."""
    B = U.shape[0]
    if cosine:
        uh, nu, fu = l2_normalize_cols(U)
        vh, nv, fv = l2_normalize_cols(V)
    else:
        uh, vh = U, V
    o = (uh * vh).sum(1)
    y = np.asarray(label, np.float64) / max_rating
    p = np.clip(o, BCE_EPS, BCE_HI)
    loss = -(y * np.log(p + BCE_EPS) + (1 - y) * np.log(1 - p + BCE_EPS)).mean()
    g = np.where((o >= BCE_EPS) & (o <= BCE_HI), -(y / (p + BCE_EPS) - (1 - y) / (1 - p + BCE_EPS)) / B, 0.0)
    duh, dvh = g[:, None] * vh, g[:, None] * uh
    if not cosine:
        return loss, duh, dvh, o
    dU = nu * (duh - fu * uh * (uh * duh).sum(0))
    dV = nv * (dvh - fv * vh * (vh * dvh).sum(0))
    return loss, dU, dV, o


def step(R, Wu, bu, Wi, bi, users, items, ratings, max_rating, cosine):
    """One train_step's loss and gradients in fp64: R is the dense train rating matrix; the user tower reads R[users],
    the item tower R.T[items].  Returns (loss, dWu, dbu, dWi, dbi, outputs, user outputs, item outputs)."""
    Xu, Xi = R[users], R.T[items]
    U, pu, au = tower(Xu, Wu, bu)
    V, pi, ai = tower(Xi, Wi, bi)
    loss, dU, dV, o = head(U, V, ratings, max_rating, cosine)
    dWu, dbu = tower_backward(Xu, Wu, pu, au, dU)
    dWi, dbi = tower_backward(Xi, Wi, pi, ai, dV)
    return loss, dWu, dbu, dWi, dbi, o, U, V


def get_recs_literal(R, Wu, bu, Wi, bi, offset, stop, cosine):
    """get_recs (model.py:119-132) on the block [offset, stop) as the reference forms it: (B, n_items) user and item index
    matrices, (B, n_items, F) tower outputs, normalised over axis 0, summed over the factors."""
    n_items = R.shape[1]
    B = stop - offset
    users = np.repeat(np.arange(offset, stop)[:, None], n_items, 1)
    items = np.array([np.arange(n_items) for _ in range(B)])
    U = tower(R[users.reshape(-1)], Wu, bu)[0].reshape(B, n_items, -1)
    V = tower(R.T[items.reshape(-1)], Wi, bi)[0].reshape(B, n_items, -1)
    if cosine:
        U = U / np.sqrt(np.maximum((U * U).sum(0, keepdims=True), L2_EPS))
        V = V / np.sqrt(np.maximum((V * V).sum(0, keepdims=True), L2_EPS))
    return (U * V).sum(-1)


def score_operands(Uo, Vo, block, cosine):
    """The factorised form eb_dmf_score_operands_f32 computes, in fp64: (U^ for every user by blocks, {block size: V^})."""
    n_users = Uo.shape[0]
    bl = min(block, n_users)
    sizes = {bl, n_users - (n_users - 1) // bl * bl}
    if not cosine:
        return Uo.copy(), {s: Vo.copy() for s in sizes}
    Uh = np.empty_like(Uo)
    for o in range(0, n_users, bl):
        blk = Uo[o:o + bl]
        Uh[o:o + bl] = blk / np.sqrt(np.maximum((blk * blk).sum(0), L2_EPS))
    return Uh, {s: Vo / np.sqrt(np.maximum(s * Vo * Vo, L2_EPS)) for s in sizes}


class Sampler:
    """Host restatement of the pointwise ratio sampler: one legacy MT19937 stream (RandomState(42)), per sample
    u = randint(n_users), the in-place shuffle of [0]*neg_ratio + [1] written out as its swaps (for i = n-1 .. 1,
    j uniform on [0, i] by the same masked rejection randint uses), then a positive rows[u][randint(len)] with its rating
    when the list's first slot holds the 1, else randint(n_items) redrawn while it is one of u's items, rating 0.
    `rows[u]` is u's item list in the order the reference iterates it, `ratings[u]` the matching ratings."""

    def __init__(self, rows, ratings, n_items, neg_ratio, seed=42):
        self.rs = np.random.RandomState(seed)
        self.rows, self.ratings, self.n_items, self.neg_ratio = rows, ratings, n_items, neg_ratio
        self.sets = [set(r) for r in rows]

    def epoch(self, events):
        rs, n = self.rs, self.neg_ratio + 1
        lst = [0] * self.neg_ratio + [1]
        out = np.empty((events, 3), np.float64)
        for t in range(events):
            u = rs.randint(len(self.rows))
            for i in range(n - 1, 0, -1):
                j = rs.randint(i + 1)
                lst[i], lst[j] = lst[j], lst[i]
            if lst[0]:
                k = rs.randint(len(self.rows[u]))
                out[t] = (u, self.rows[u][k], self.ratings[u][k])
            else:
                it = rs.randint(self.n_items)
                while it in self.sets[u]:
                    it = rs.randint(self.n_items)
                out[t] = (u, it, 0.0)
        return out[:, 0].astype(np.int32), out[:, 1].astype(np.int32), out[:, 2].astype(np.float32)
