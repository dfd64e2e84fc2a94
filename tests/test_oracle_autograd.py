"""The hand-derived gradients of the TensorFlow-model restatements (oracle/tf_models.py, parity unpinned against TF itself)
checked against an independent automatic differentiation of the SAME forward formulas written with torch ops in
fp64 on the CPU (the formulas follow the reference's model code: BPRMF_batch_model.py:46-75,
multi_vae_model.py:114-142, neural_matrix_factorization_model.py:74-106).  This does not pin the restatements to a
TensorFlow run — it rules out algebra mistakes in the backward passes the GPU kernels are tested against."""
import numpy as np
import torch

from oracle import tf_models as tfm

T = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)


def test_bprmf_batch_gradients_match_autograd():
    rs = np.random.RandomState(0)
    nu, ni, d, B = 30, 40, 6, 200
    Gu, Gi, Bi = rs.normal(0, 0.3, (nu, d)), rs.normal(0, 0.3, (ni, d)), rs.normal(0, 0.1, ni)
    u, i, j = rs.randint(nu, size=B), rs.randint(ni, size=B), rs.randint(ni, size=B)
    l_w, l_b = 0.1, 0.001
    loss, dGu, dGi, dBi = tfm.bprmf_batch_loss_and_grads(Gu, Gi, Bi, u, i, j, l_w, l_b)
    tGu, tGi, tBi = T(Gu), T(Gi), T(Bi)
    gu, gp, gn, bp, bn = tGu[u], tGi[i], tGi[j], tBi[i], tBi[j]
    diff = torch.clamp((bp + (gu * gp).sum(1)) - (bn + (gu * gn).sum(1)), -80.0, 1e8)
    tl = torch.nn.functional.softplus(-diff).sum() + l_w * ((gu ** 2).sum() / 2 + (gp ** 2).sum() / 2 + (gn ** 2).sum() / 2) \
        + l_b * (bp ** 2).sum() / 2 + l_b * (bn ** 2).sum() / 2 / 10
    tl.backward()
    assert abs(tl.item() - loss) < 1e-10 * abs(loss)
    for a, b in ((dGu, tGu.grad), (dGi, tGi.grad), (dBi, tBi.grad)):
        assert np.abs(a - b.numpy()).max() < 1e-12


def _dropout_mask(rs, shape, rate):
    """(keep mask, rate) of Keras Dropout at `rate`, or (None, 0) for no dropout."""
    return (None, 0.0) if rate == 0 else ((rs.rand(*shape) >= rate).astype(np.float64), rate)


def _dropped(xh, keep, rate):
    return xh if keep is None else xh * torch.tensor(keep) / (1.0 - rate)


def test_multivae_gradients_match_autograd():
    _check_multivae(0.0)


def test_multivae_dropout_gradients_match_autograd():
    """The same with the input dropout of dropout_pkeep = 0.5 (a fixed keep mask, Keras 1/(1-rate) scale)."""
    _check_multivae(0.5)


def _check_multivae(rate):
    rs = np.random.RandomState(1)
    B, I, H, L = 12, 50, 16, 8
    P = {"W1": rs.normal(0, 0.2, (I, H)), "b1": rs.normal(0, 0.05, H), "W2": rs.normal(0, 0.2, (H, 2 * L)), "b2": rs.normal(0, 0.05, 2 * L),
         "W3": rs.normal(0, 0.2, (L, H)), "b3": rs.normal(0, 0.05, H), "W4": rs.normal(0, 0.2, (H, I)), "b4": rs.normal(0, 0.05, I)}
    X = (rs.rand(B, I) < 0.2).astype(np.float64); X[0] = 0; X[0, 3] = 1
    eps = rs.normal(size=(B, L)); anneal = 0.17
    keep, rate = _dropout_mask(rs, (B, I), rate)
    loss, G, _ = tfm.multivae_forward_backward(P, X, eps, anneal, keep=keep, rate=rate)
    tp = {k: T(v) for k, v in P.items()}
    tx, te = torch.tensor(X), torch.tensor(eps)
    xh = _dropped(torch.nn.functional.normalize(tx, p=2, dim=1), keep, rate)       # tf.nn.l2_normalize, then Dropout
    h1 = torch.tanh(xh @ tp["W1"] + tp["b1"])
    ml = h1 @ tp["W2"] + tp["b2"]
    mu, lv = ml[:, :L], ml[:, L:]
    z = mu + torch.exp(0.5 * lv) * te
    logits = torch.tanh(z @ tp["W3"] + tp["b3"]) @ tp["W4"] + tp["b4"]
    kl = -0.5 * torch.mean(lv - mu ** 2 - torch.exp(lv) + 1)
    nll = -torch.mean((torch.log_softmax(logits, 1) * tx).sum(1))
    tl = nll + anneal * kl
    tl.backward()
    assert abs(tl.item() - loss) < 1e-12 * abs(loss)
    for k in P:
        assert np.abs(G[k] - tp[k].grad.numpy()).max() < 1e-12, k


def test_neumf_gradients_match_autograd():
    rs = np.random.RandomState(2)
    nu, ni, f, B = 20, 25, 4, 64
    P = {"U_mf": rs.normal(0, 0.3, (nu, f)), "I_mf": rs.normal(0, 0.3, (ni, f)), "U_mlp": rs.normal(0, 0.3, (nu, f)),
         "I_mlp": rs.normal(0, 0.3, (ni, f)), "W1": rs.normal(0, 0.3, (2 * f, 4 * f)), "b1": rs.normal(0, 0.1, 4 * f),
         "W2": rs.normal(0, 0.3, (4 * f, 2 * f)), "b2": rs.normal(0, 0.1, 2 * f), "W3": rs.normal(0, 0.3, (2 * f, f)),
         "b3": rs.normal(0, 0.1, f), "wp": rs.normal(0, 0.3, 2 * f), "bp": np.array(0.05)}
    u, i = rs.randint(nu, size=B), rs.randint(ni, size=B)
    y = (rs.rand(B) < 0.4).astype(np.float64)
    loss, G, _ = tfm.neumf_forward_backward(P, u, i, y)
    tp = {k: T(v) for k, v in P.items()}
    x0 = torch.cat([tp["U_mlp"][u], tp["I_mlp"][i]], 1)
    h = torch.relu(x0 @ tp["W1"] + tp["b1"]); h = torch.relu(h @ tp["W2"] + tp["b2"]); h = torch.relu(h @ tp["W3"] + tp["b3"])
    logit = torch.cat([tp["U_mf"][u] * tp["I_mf"][i], h], 1) @ tp["wp"] + tp["bp"]
    p = torch.clamp(torch.sigmoid(logit), 1e-7, 1 - 1e-7)
    ty = torch.tensor(y)
    tl = torch.mean(-(ty * torch.log(p) + (1 - ty) * torch.log(1 - p)))
    tl.backward()
    assert abs(tl.item() - loss) < 1e-12 * abs(loss)
    for k in P:
        assert np.abs(np.asarray(G[k]) - tp[k].grad.numpy()).max() < 1e-12, k


def test_multidae_gradients_match_autograd():
    _check_multidae(0.0)


def test_multidae_dropout_gradients_match_autograd():
    _check_multidae(0.2)


def _check_multidae(rate):
    rs = np.random.RandomState(3)
    B, I, H, L = 10, 40, 16, 8
    P = {"W1": rs.normal(0, 0.2, (I, H)), "b1": rs.normal(0, 0.05, H), "W2": rs.normal(0, 0.2, (H, L)), "b2": rs.normal(0, 0.05, L),
         "W3": rs.normal(0, 0.2, (L, H)), "b3": rs.normal(0, 0.05, H), "W4": rs.normal(0, 0.2, (H, I)), "b4": rs.normal(0, 0.05, I)}
    X = (rs.rand(B, I) < 0.2).astype(np.float64); X[0] = 0; X[0, 3] = 1
    keep, rate = _dropout_mask(rs, (B, I), rate)
    loss, G, _ = tfm.multidae_forward_backward(P, X, keep=keep, rate=rate)
    tp = {k: T(v) for k, v in P.items()}
    tx = torch.tensor(X)
    xh = _dropped(torch.nn.functional.normalize(tx, p=2, dim=1), keep, rate)
    h = torch.tanh(xh @ tp["W1"] + tp["b1"]); h = torch.tanh(h @ tp["W2"] + tp["b2"]); h = torch.tanh(h @ tp["W3"] + tp["b3"])
    tl = -torch.mean((torch.log_softmax(h @ tp["W4"] + tp["b4"], 1) * tx).sum(1))
    tl.backward()
    assert abs(tl.item() - loss) < 1e-12 * abs(loss)
    for k in P:
        assert np.abs(G[k] - tp[k].grad.numpy()).max() < 1e-12, k


def test_gmf_gradients_match_autograd():
    rs = np.random.RandomState(4)
    nu, ni, f, B = 20, 25, 6, 80
    P = {"U": rs.normal(0, 0.4, (nu, f)), "I": rs.normal(0, 0.4, (ni, f)), "h": rs.normal(0, 0.5, f)}
    u, i = rs.randint(nu, size=B), rs.randint(ni, size=B)
    y = (rs.rand(B) < 0.5).astype(np.float64)
    loss, G, _ = tfm.gmf_forward_backward(P, u, i, y)
    tp = {k: T(v) for k, v in P.items()}
    p = torch.clamp(torch.sigmoid((tp["U"][u] * tp["I"][i]) @ tp["h"]), 1e-7, 1 - 1e-7)
    ty = torch.tensor(y)
    tl = torch.mean(-(ty * torch.log(p) + (1 - ty) * torch.log(1 - p)))
    tl.backward()
    assert abs(tl.item() - loss) < 1e-12 * abs(loss)
    for k in P:
        assert np.abs(G[k] - tp[k].grad.numpy()).max() < 1e-12, k


def test_keras_adam_restatement_first_steps():
    """KerasAdam against the closed form of its own first steps (lr_t, epsilon placement as documented for TF 2.3)."""
    opt = tfm.KerasAdam(0.01)
    var = np.array([1.0, -2.0]); g = np.array([0.5, -0.25])
    opt.begin_step(); opt.apply("v", var, g)
    lr_t = 0.01 * np.sqrt(1 - 0.999) / (1 - 0.9)
    want = np.array([1.0, -2.0]) - lr_t * (0.1 * g) / (np.sqrt(0.001 * g * g) + 1e-7)
    assert np.allclose(var, want, rtol=0, atol=1e-15)
