"""fp64 NumPy restatements of the reference's TensorFlow models.  TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED: tensorflow==2.3.2 (requirements.txt:3) is absent from the build container and
its source is not part of the original project, so these follow the reference's model code line by
line plus the published TF 2.3 semantics they rely on (stated per function).  Nothing here was
checked against a TensorFlow run.  What IS checked: the backward passes against an independent fp64 autodiff of the
same forward formulas (tests/test_oracle_autograd.py).
"""
import numpy as np


def softplus(x):
    return np.where(x > 0, x + np.log1p(np.exp(-np.abs(x))), np.log1p(np.exp(-np.abs(x))))


def bprmf_batch_loss_and_grads(Gu, Gi, Bi, u, i, j, l_w, l_b):
    """BPRMF_batch_model.call/train_step, BPRMF_batch_model.py:46-75.
    TF semantics assumed: tf.nn.l2_loss(t) = sum(t**2)/2 over the gathered batch rows;
    clip_by_value passes gradient only strictly inside (-80, 1e8); gradients w.r.t. the
    variables are IndexedSlices whose duplicate indices are summed when applied."""
    gu, gp, gn = Gu[u], Gi[i], Gi[j]
    bp, bn = Bi[i], Bi[j]
    raw = (bp + (gu * gp).sum(1)) - (bn + (gu * gn).sum(1))
    diff = np.clip(raw, -80.0, 1e8)
    loss = softplus(-diff).sum() + l_w * ((gu ** 2).sum() + (gp ** 2).sum() + (gn ** 2).sum()) / 2 \
        + l_b * (bp ** 2).sum() / 2 + l_b * (bn ** 2).sum() / 2 / 10
    g = np.where((raw > -80.0) & (raw < 1e8), -1.0 / (1.0 + np.exp(diff)), 0.0)
    dGu = np.zeros_like(Gu); dGi = np.zeros_like(Gi); dBi = np.zeros_like(Bi)
    np.add.at(dGu, u, g[:, None] * (gp - gn) + l_w * gu)
    np.add.at(dGi, i, g[:, None] * gu + l_w * gp)
    np.add.at(dGi, j, -g[:, None] * gu + l_w * gn)
    np.add.at(dBi, i, g + l_b * bp)
    np.add.at(dBi, j, -g + l_b * bn / 10)
    return loss, dGu, dGi, dBi


class KerasAdam:
    """tf.optimizers.Adam(lr) as used at BPRMF_batch_model.py:44,77-78.  TF 2.3 OptimizerV2 Adam:
    beta_1=0.9, beta_2=0.999, epsilon=1e-7, lr_t = lr*sqrt(1-b2^t)/(1-b1^t); the sparse apply
    decays m and v and updates the variable for EVERY row (dense-equivalent with the summed
    IndexedSlices gradient)."""

    def __init__(self, lr, b1=0.9, b2=0.999, eps=1e-7):
        self.lr, self.b1, self.b2, self.eps, self.t = lr, b1, b2, eps, 0
        self.state = {}

    def begin_step(self):
        self.t += 1

    def apply(self, name, var, grad):
        m, v = self.state.setdefault(name, (np.zeros_like(var), np.zeros_like(var)))
        lr_t = self.lr * np.sqrt(1 - self.b2 ** self.t) / (1 - self.b1 ** self.t)
        m *= self.b1; m += (1 - self.b1) * grad
        v *= self.b2; v += (1 - self.b2) * grad * grad
        var -= lr_t * m / (np.sqrt(v) + self.eps)


def bprmf_batch_step(Gu, Gi, Bi, opt, u, i, j, l_w, l_b):
    loss, dGu, dGi, dBi = bprmf_batch_loss_and_grads(Gu, Gi, Bi, u, i, j, l_w, l_b)
    opt.begin_step()
    opt.apply("Bi", Bi, dBi); opt.apply("Gu", Gu, dGu); opt.apply("Gi", Gi, dGi)
    return loss


def glorot_uniform(rng, shape):
    """tf.initializers.GlorotUniform limits (values come from TF's own Philox stream, which
    cannot be replayed here)."""
    lim = np.sqrt(6.0 / (shape[0] + shape[1]))
    return rng.uniform(-lim, lim, size=shape)


# ---------------------------------------------------------------- MultiVAE (parity unpinned)
def _dropout_input(X, keep, rate):
    """l2_normalize (multi_vae_model.py:42) then Keras Dropout (:43): kept entries scaled by 1/(1-rate), `keep` the 0/1 mask
    (None: no dropout)."""
    nrm = np.sqrt((X ** 2).sum(1, keepdims=True)); nrm[nrm == 0] = 1.0
    xh = X / nrm
    return xh if keep is None else xh * keep / (1.0 - rate)


def multivae_forward_backward(P, X, eps, anneal, keep=None, rate=0.0):
    """VariationalAutoEncoder.call/train_step, multi_vae_model.py:114-142, for a dense binary batch X
    (B x I) and given reparametrisation noise eps (B x L).  P holds Keras-layout weights:
    W1 (I x H), b1, W2 (H x 2L: dense_mean | dense_log_var), b2, W3 (L x H), b3, W4 (H x I), b4.
    keep (B x I, 0/1) with rate: the input dropout mask, applied after l2_normalize with the 1/(1-rate) scale.
    kernel_regularizer losses are declared but never added to the loss in the reference
    (multi_vae_model.py:47-53,75-78 vs :136) -> reg_lambda is inert, as here.
    Returns loss, grads dict, (logits, mu, lv, z)."""
    B, L = eps.shape
    xh = _dropout_input(X, keep, rate)
    h1 = np.tanh(xh @ P["W1"] + P["b1"])
    ml = h1 @ P["W2"] + P["b2"]
    mu, lv = ml[:, :L], ml[:, L:]
    z = mu + np.exp(0.5 * lv) * eps                               # Sampling, :20-29
    h2 = np.tanh(z @ P["W3"] + P["b3"])
    logits = h2 @ P["W4"] + P["b4"]
    m = logits.max(1, keepdims=True)
    lse = m + np.log(np.exp(logits - m).sum(1, keepdims=True))
    ls = logits - lse
    kl = -0.5 * np.mean(lv - mu ** 2 - np.exp(lv) + 1)            # :119-121
    neg_ll = -np.mean((ls * X).sum(1))                            # :131-135
    loss = neg_ll + anneal * kl
    dlogits = (np.exp(ls) * X.sum(1, keepdims=True) - X) / B
    G = {"W4": h2.T @ dlogits, "b4": dlogits.sum(0)}
    dpre2 = (dlogits @ P["W4"].T) * (1 - h2 ** 2)
    G["W3"] = z.T @ dpre2; G["b3"] = dpre2.sum(0)
    dz = dpre2 @ P["W3"].T
    dmu = dz + anneal * mu / (B * L)
    dlv = dz * 0.5 * np.exp(0.5 * lv) * eps + anneal * 0.5 * (np.exp(lv) - 1) / (B * L)
    dml = np.concatenate([dmu, dlv], 1)
    G["W2"] = h1.T @ dml; G["b2"] = dml.sum(0)
    dpre1 = (dml @ P["W2"].T) * (1 - h1 ** 2)
    G["W1"] = xh.T @ dpre1; G["b1"] = dpre1.sum(0)
    return loss, G, (logits, mu, lv, z, neg_ll, kl)


# Keras BinaryCrossentropy clips fp32 probabilities to [epsilon, 1 - epsilon] with epsilon = 1e-7 as fp32 constants: the
# upper bound is 1 - 2^-23 (0.99999988), which sets the loss of a saturated sample (-log(1.19e-7), not -log(1e-7))
CLIP_LO, CLIP_HI = float(np.float32(1e-7)), float(np.float32(1.0) - np.float32(1e-7))


def _bce_clip(p, y):
    """(mean-reduction numerator terms, d loss / d logit numerators) of Keras BinaryCrossentropy on probabilities p"""
    pc = np.clip(p, CLIP_LO, CLIP_HI)
    return -(y * np.log(pc) + (1 - y) * np.log(1 - pc)), np.where((p > CLIP_LO) & (p < CLIP_HI), p - y, 0.0)


# ---------------------------------------------------------------- NeuMF (parity unpinned)
def neumf_forward_backward(P, u, i, y):
    """NeuralMatrixFactorizationModel.call/train_step (neural_matrix_factorization_model.py:74-106), dropout 0,
    is_mf_train = is_mlp_train = True.  P: U_mf, I_mf, U_mlp, I_mlp (tables), W1 (2f x 4f), b1, W2 (4f x 2f), b2,
    W3 (2f x f), b3, wp (2f), bp (scalar) in Keras layout.  Keras BinaryCrossentropy: mean over the batch of
    -(y log p + (1-y) log(1-p)) with p clipped to [CLIP_LO, CLIP_HI]."""
    B = len(u)
    x0 = np.concatenate([P["U_mlp"][u], P["I_mlp"][i]], 1)
    pm = P["U_mf"][u] * P["I_mf"][i]
    h1 = np.maximum(x0 @ P["W1"] + P["b1"], 0); h2 = np.maximum(h1 @ P["W2"] + P["b2"], 0)
    h3 = np.maximum(h2 @ P["W3"] + P["b3"], 0)
    feat = np.concatenate([pm, h3], 1)
    logit = feat @ P["wp"] + P["bp"]
    p = 1 / (1 + np.exp(-logit))
    bce, g = _bce_clip(p, y)
    loss = np.mean(bce)
    dl = g / B
    f = pm.shape[1]
    G = {"wp": feat.T @ dl, "bp": dl.sum()}
    dpm = dl[:, None] * P["wp"][None, :f]
    dpre3 = (dl[:, None] * P["wp"][None, f:]) * (h3 > 0)
    G["W3"] = h2.T @ dpre3; G["b3"] = dpre3.sum(0)
    dpre2 = (dpre3 @ P["W3"].T) * (h2 > 0)
    G["W2"] = h1.T @ dpre2; G["b2"] = dpre2.sum(0)
    dpre1 = (dpre2 @ P["W2"].T) * (h1 > 0)
    G["W1"] = x0.T @ dpre1; G["b1"] = dpre1.sum(0)
    dx0 = dpre1 @ P["W1"].T
    for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
        G[k] = np.zeros_like(P[k])
    np.add.at(G["U_mf"], u, dpm * P["I_mf"][i]); np.add.at(G["I_mf"], i, dpm * P["U_mf"][u])
    np.add.at(G["U_mlp"], u, dx0[:, :f]); np.add.at(G["I_mlp"], i, dx0[:, f:])
    return loss, G, p


# ---------------------------------------------------------------- MultiDAE (parity unpinned)
def multidae_forward_backward(P, X, keep=None, rate=0.0):
    """DenoisingAutoEncoder.call/train_step (autoencoders/dae/multi_dae_model.py:20-125): l2-normalised rows -> input
    dropout (keep mask with rate, as multivae_forward_backward; None: dropout 0) -> tanh Dense(I->H) -> tanh Dense(H->L)
    -> tanh Dense(L->H) -> Dense(H->I); loss = -mean_u sum_i log_softmax * x.
    P in Keras layout: W1 (I x H), b1, W2 (H x L), b2, W3 (L x H), b3, W4 (H x I), b4.  Returns loss, grads, logits."""
    B = X.shape[0]
    xh = _dropout_input(X, keep, rate)
    h1 = np.tanh(xh @ P["W1"] + P["b1"])
    zm = np.tanh(h1 @ P["W2"] + P["b2"])
    h2 = np.tanh(zm @ P["W3"] + P["b3"])
    logits = h2 @ P["W4"] + P["b4"]
    m = logits.max(1, keepdims=True)
    ls = logits - (m + np.log(np.exp(logits - m).sum(1, keepdims=True)))
    loss = -np.mean((ls * X).sum(1))
    dlogits = (np.exp(ls) * X.sum(1, keepdims=True) - X) / B
    G = {"W4": h2.T @ dlogits, "b4": dlogits.sum(0)}
    dpre2 = (dlogits @ P["W4"].T) * (1 - h2 ** 2)
    G["W3"] = zm.T @ dpre2; G["b3"] = dpre2.sum(0)
    dprez = (dpre2 @ P["W3"].T) * (1 - zm ** 2)
    G["W2"] = h1.T @ dprez; G["b2"] = dprez.sum(0)
    dpre1 = (dprez @ P["W2"].T) * (1 - h1 ** 2)
    G["W1"] = xh.T @ dpre1; G["b1"] = dpre1.sum(0)
    return loss, G, logits


# ---------------------------------------------------------------- GMF (parity unpinned)
def gmf_forward_backward(P, u, i, y):
    """GeneralizedMatrixFactorizationModel.call/train_step (generalized_matrix_factorization_model.py:56-75),
    is_edge_weight_train = True: p = sigmoid((U[u]*I[i]) @ h), Keras BinaryCrossentropy (batch mean, p clipped to
    [CLIP_LO, CLIP_HI]).  P: U, I (tables), h (f).  Returns loss, grads, p."""
    B = len(u)
    pm = P["U"][u] * P["I"][i]
    p = 1 / (1 + np.exp(-(pm @ P["h"])))
    bce, g = _bce_clip(p, y)
    loss = np.mean(bce)
    dl = g / B
    G = {"h": pm.T @ dl, "U": np.zeros_like(P["U"]), "I": np.zeros_like(P["I"])}
    dpm = dl[:, None] * P["h"][None, :]
    np.add.at(G["U"], u, dpm * P["I"][i]); np.add.at(G["I"], i, dpm * P["U"][u])
    return loss, G, p
