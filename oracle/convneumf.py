"""fp64 NumPy restatements of the reference's ConvNeuMF (neural/ConvNeuMF/convolutional_neural_matrix_factorization_model.py).
TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED, as for every TensorFlow model here (oracle/tf_models.py): the restatement follows the model code plus the
TF 2.3 semantics it relies on:
  - the sampler's [B, 1] columns make the embeddings [B, 1, f], so matmul(u, i, transpose_a=True) is the outer product
    M[x][y] = u[x] i[y] (rows from the user), expanded to [B, f, f, 1] (:114-116);
  - Conv2D(k, c, strides=s, 'valid', relu) per layer, kernels [kh][kw][c_in][c_out]; reduce_sum over both spatial axes
    (:118); Dropout -> Dense(c_L) -> Dropout -> Dense(1), both linear (:47-66);
  - loss = sum softplus(-clip(x+ - x-, -80, 1e8)) + l_w (l2_loss(u) + l2_loss(i) + l2_loss(j)), l2_loss(t) = sum(t^2)/2;
    the clip passes the gradient strictly inside (-80, 1e8) (the convention of oracle/tf_models.py); Keras Adam is
    tf_models.KerasAdam.

Parameters are a dict in Keras shapes: W1 [2,2,1,c1], b1, K[l] [2,2,c_(l-1),c_l] and b[l] for l >= 2 (lists indexed by
level, entries 0 and 1 unused), Wd1 [cL,cL], bd1 [cL], wd2 [cL], bd2 [1].

Two forward forms: `literal_forward`, the map and its convolutions as the reference forms them, and `quadtree_forward`,
the Z-order GEMM form of csrc/convneumf.cu (level 1 from S, levels >= 2 as [rows_l][4 c_(l-1)] x [4 c_(l-1)][c_l]).
`loss_and_grads` is the hand-written backward of the quad-tree form; tests/test_oracle_convneumf.py checks both forms
against torch (conv2d and autograd)."""
import numpy as np

from .tf_models import KerasAdam  # noqa: F401  (re-exported: the optimiser these tests step)

CLIP_LO, CLIP_HI = -80.0, 1e8


def geometry(f, L):
    """(H_L, m): final positions per axis and the embedding coordinates the network reads."""
    HL = f >> L
    return HL, HL << L


def glorot_limits(channels):
    """GlorotUniform limits sqrt(6 / (fan_in + fan_out)) of W1, K[2..L] and Wd1, wd2 (conv fans k^2 c_in, k^2 c_out)."""
    c = list(channels)
    lims = {"W1": np.sqrt(6.0 / (4 * 1 + 4 * c[0]))}
    for l in range(2, len(c) + 1):
        lims[f"K{l}"] = np.sqrt(6.0 / (4 * c[l - 2] + 4 * c[l - 1]))
    lims["Wd1"] = np.sqrt(6.0 / (2 * c[-1]))
    lims["wd2"] = np.sqrt(6.0 / (c[-1] + 1))
    return lims


def init_params(rng, channels, scale=1.0):
    """Random parameters (GlorotUniform limits, biases drawn too so that every path is exercised), Keras shapes."""
    c = [1] + list(channels)
    L = len(channels)
    lim = glorot_limits(channels)
    P = {"W1": rng.uniform(-lim["W1"], lim["W1"], (2, 2, 1, c[1])) * scale, "b1": rng.uniform(-0.05, 0.05, c[1]),
         "K": [None, None] + [rng.uniform(-lim[f"K{l}"], lim[f"K{l}"], (2, 2, c[l - 1], c[l])) * scale for l in range(2, L + 1)],
         "b": [None, None] + [rng.uniform(-0.05, 0.05, c[l]) for l in range(2, L + 1)],
         "Wd1": rng.uniform(-lim["Wd1"], lim["Wd1"], (c[L], c[L])), "bd1": rng.uniform(-0.05, 0.05, c[L]),
         "wd2": rng.uniform(-lim["wd2"], lim["wd2"], c[L]), "bd2": rng.uniform(-0.05, 0.05, 1)}
    return P


def head(P, s, m1=None, m2=None):
    """Dropout -> Dense(cL) -> Dropout -> Dense(1) on the summed last level s [B, cL]; m1 / m2 the dropout scales."""
    x1 = s if m1 is None else s * m1
    z = x1 @ P["Wd1"] + P["bd1"]
    x2 = z if m2 is None else z * m2
    return x2 @ P["wd2"] + P["bd2"][0], (x1, z, x2)


def literal_forward(P, u, i, m1=None, m2=None):
    """The reference's call() for pairs (u [B, f], i [B, f]): the [B, f, f, 1] map through every Conv2D, the spatial sum and
    the head.  Returns (y [B], the last conv level [B, H_L, H_L, c_L])."""
    x = (u[:, :, None] * i[:, None, :])[..., None]
    kernels = [(P["W1"], P["b1"])] + [(P["K"][l], P["b"][l]) for l in range(2, len(P["K"]))]
    for K, b in kernels:
        H = x.shape[1] // 2
        out = np.zeros((x.shape[0], H, H, K.shape[3])) + b
        for kh in range(2):
            for kw in range(2):
                out += np.einsum("bpqc,cd->bpqd", x[:, kh:kh + 2 * H:2, kw:kw + 2 * H:2, :], K[kh, kw])
        x = np.maximum(out, 0.0)
    y, _ = head(P, x.sum(axis=(1, 2)), m1, m2)
    return y, x


def zorder(HL, lr):
    """(a, b) of every local row of a level with lr = L - l low bit pairs, in Z-order (csrc/convneumf.cu)."""
    R = HL * HL << (2 * lr)
    r = np.arange(R)
    t, rem = r >> (2 * lr), r & ((1 << (2 * lr)) - 1)
    da = np.zeros(R, np.int64); db = np.zeros(R, np.int64)
    for k in range(lr):
        da |= ((rem >> (2 * k + 1)) & 1) << k
        db |= ((rem >> (2 * k)) & 1) << k
    return (t // HL) << lr | da, (t % HL) << lr | db


def level1(P, u, i, L):
    """Level-1 pre-activations [B, R_1, c1] in Z-order from S0 / S1 (the bilinear form)."""
    f = u.shape[1]
    HL, _ = geometry(f, L)
    a, b = zorder(HL, L - 1)
    W = P["W1"][:, :, 0, :]                                        # [da][db][c]
    S0 = u[:, 2 * a, None] * W[0, 0] + u[:, 2 * a + 1, None] * W[1, 0]
    S1 = u[:, 2 * a, None] * W[0, 1] + u[:, 2 * a + 1, None] * W[1, 1]
    return S0 * i[:, 2 * b, None] + S1 * i[:, 2 * b + 1, None] + P["b1"]


def quadtree_forward(P, u, i, m1=None, m2=None):
    """The same network in the Z-order GEMM form: (y [B], [h_1 .. h_L] relu'd levels [B, R_l, c_l], head values)."""
    L = len(P["K"]) - 1
    h = [None, np.maximum(level1(P, u, i, L), 0.0)]
    for l in range(2, L + 1):
        K = P["K"][l]
        X = h[-1].reshape(h[-1].shape[0], -1, 4 * K.shape[2])
        h.append(np.maximum(X @ K.reshape(4 * K.shape[2], K.shape[3]) + P["b"][l], 0.0))
    y, hv = head(P, h[L].sum(axis=1), m1, m2)
    return y, h, hv


def _backward_pairs(P, u, i, h, hv, dy, m1, m2, G):
    """Adds the parameter gradients of pairs (u, i) with upstream dy [B] to G; returns (du [B, f], di [B, f])."""
    L = len(P["K"]) - 1
    x1, z, x2 = hv
    G["wd2"] += x2.T @ dy
    G["bd2"] += dy.sum()
    dz = dy[:, None] * P["wd2"][None, :]
    if m2 is not None:
        dz = dz * m2
    G["Wd1"] += x1.T @ dz
    G["bd1"] += dz.sum(0)
    ds = dz @ P["Wd1"].T
    if m1 is not None:
        ds = ds * m1
    d = ds[:, None, :] * (h[L] > 0)
    for l in range(L, 1, -1):
        K = P["K"][l]
        cin = K.shape[2]
        X = h[l - 1].reshape(h[l - 1].shape[0], -1, 4 * cin)
        G["K"][l] += np.einsum("brk,brn->kn", X, d).reshape(K.shape)
        G["b"][l] += d.sum(axis=(0, 1))
        dX = d @ K.reshape(4 * cin, K.shape[3]).T
        d = dX.reshape(h[l - 1].shape) * (h[l - 1] > 0)
    f = u.shape[1]
    HL, m = geometry(f, L)
    A = m // 2
    a, b = zorder(HL, L - 1)
    g = np.zeros((d.shape[0], A, A, d.shape[2]))
    g[:, a, b, :] = d
    W = P["W1"][:, :, 0, :]
    ur, ir = u[:, :m].reshape(-1, A, 2), i[:, :m].reshape(-1, A, 2)          # [n][a][da], [n][b][db]
    G["W1"][:, :, 0, :] += np.einsum("nabc,nax,nby->xyc", g, ur, ir)
    G["b1"] += g.sum(axis=(0, 1, 2))
    du = np.zeros_like(u); di = np.zeros_like(i)
    du[:, :m] = np.einsum("nabc,xyc,nby->nax", g, W, ir).reshape(-1, m)
    di[:, :m] = np.einsum("nabc,xyc,nax->nby", g, W, ur).reshape(-1, m)
    return du, di


def zero_grads(P):
    return {k: ([None if t is None else np.zeros_like(t) for t in v] if isinstance(v, list) else np.zeros_like(v))
            for k, v in P.items()}


def loss_and_grads(P, U, I, tu, ti, tj, l_w, masks=None):
    """The reference's train_step loss and every gradient for triples (tu, ti, tj): (loss, G, dU, dI, (y+, y-)).
    masks: None (dropout off) or (m1+, m2+, m1-, m2-) dropout scales [B, cL] of the positive and negative pairs."""
    m1p, m2p, m1n, m2n = masks if masks is not None else (None,) * 4
    u, i, j = U[tu], I[ti], I[tj]
    yp, hp, hvp = quadtree_forward(P, u, i, m1p, m2p)
    yn, hn, hvn = quadtree_forward(P, u, j, m1n, m2n)
    x = yp - yn
    xc = np.clip(x, CLIP_LO, CLIP_HI)
    loss = np.logaddexp(0.0, -xc).sum() + l_w * ((u ** 2).sum() + (i ** 2).sum() + (j ** 2).sum()) / 2
    g = np.where((x > CLIP_LO) & (x < CLIP_HI), -1.0 / (1.0 + np.exp(xc)), 0.0)
    G = zero_grads(P)
    du_p, di_p = _backward_pairs(P, u, i, hp, hvp, g, m1p, m2p, G)
    du_n, dj_n = _backward_pairs(P, u, j, hn, hvn, -g, m1n, m2n, G)
    dU = np.zeros_like(U); dI = np.zeros_like(I)
    np.add.at(dU, tu, du_p + du_n + l_w * u)
    np.add.at(dI, ti, di_p + l_w * i)
    np.add.at(dI, tj, dj_n + l_w * j)
    return loss, G, dU, dI, (yp, yn)


def adam_step(opt, P, U, I, G, dU, dI):
    """One Keras Adam step over every trainable weight (the embeddings, the conv kernels and biases, the head)."""
    opt.begin_step()
    opt.apply("U", U, dU); opt.apply("I", I, dI)
    opt.apply("W1", P["W1"], G["W1"]); opt.apply("b1", P["b1"], G["b1"])
    for l in range(2, len(P["K"])):
        opt.apply(f"K{l}", P["K"][l], G["K"][l]); opt.apply(f"b{l}", P["b"][l], G["b"][l])
    for k in ("Wd1", "bd1", "wd2", "bd2"):
        opt.apply(k, P[k], G[k])


def full_scores(P, U, I, users=None, block=256):
    """get_recs (:158-183) of users x every item with dropout off: [n_users, n_items] fp64, the quad-tree form."""
    users = np.arange(U.shape[0]) if users is None else np.asarray(users)
    out = np.empty((len(users), I.shape[0]))
    for r, uid in enumerate(users):
        for s in range(0, I.shape[0], block):
            e = min(s + block, I.shape[0])
            out[r, s:e] = quadtree_forward(P, np.repeat(U[uid][None], e - s, 0), I[s:e])[0]
    return out
