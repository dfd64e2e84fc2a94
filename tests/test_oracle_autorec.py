"""CPU checks of oracle/autorec.py: the fp64 step against torch autograd (both decoder activations, empty rows), the
factorised scoring against the literal get_recommendations restatements (ItemAutoRec under a non-identity
permutation), and the replay of the models' `random` calls against the sparse_sampler goldens."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import autorec

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _binary(rs, n, m, density):
    X = (rs.rand(n, m) < density).astype(np.float64)
    return X


def _weights(rs, n_in, H, n_out, scale=0.3):
    b1, b2 = autorec.init_biases(H, n_out)
    return rs.normal(0, scale, (n_in, H)), b1 + rs.normal(0, 0.1, H), rs.normal(0, scale, (H, n_out)), b2 + rs.normal(0, 0.1, n_out)


def _autograd(X, W1, b1, W2, b2, act):
    t = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)
    P = [t(W1), t(b1), t(W2), t(b2)]
    x = torch.tensor(X)
    h = torch.sigmoid(x @ P[0] + P[1])
    o = h @ P[2] + P[3]
    rec = torch.sigmoid(o) if act == "sigmoid" else o
    loss = ((x - rec * torch.sign(x)) ** 2).sum(1).mean()             # userautorec_model.py:99-102
    loss.backward()
    return loss.item(), [p.grad.numpy() for p in P]


@pytest.mark.parametrize("act", ["linear", "sigmoid"])
@pytest.mark.parametrize("B,H", [(1, 4), (7, 12), (64, 32)])
def test_step_matches_autograd(act, B, H):
    rs = np.random.RandomState(B + H)
    n = 23
    X = _binary(rs, B, n, 0.3)
    if B > 1:
        X[1] = 0.0                                                     # an empty row: counted in the mean, no gradient
    W1, b1, W2, b2 = _weights(rs, n, H, n)
    got = autorec.step(X, W1, b1, W2, b2, act)
    loss, grads = _autograd(X, W1, b1, W2, b2, act)
    assert got[0] == pytest.approx(loss, rel=1e-12)
    for a, b in zip(got[1:], grads):
        assert np.allclose(a, b, rtol=1e-10, atol=1e-14)


def test_init_biases_are_ones():
    b1, b2 = autorec.init_biases(5, 9)
    assert (b1 == 1).all() and (b2 == 1).all() and b1.shape == (5,) and b2.shape == (9,)


@pytest.mark.parametrize("block", [5, 100])
def test_user_factorised_scoring_matches_literal(block):
    rs = np.random.RandomState(block)
    nu, ni, H, k = 17, 30, 8, 6
    X = _binary(rs, nu, ni, 0.3)
    W1, b1, W2, b2 = _weights(rs, ni, H, ni)
    mask = X == 0
    v, i = autorec.get_recommendations_user(X, W1, b1, W2, b2, mask, k, block)
    h, V, b = autorec.user_scores(X, W1, b1, W2, b2)
    s = np.where(mask, h @ V.T + b, -np.inf)
    assert np.allclose(np.take_along_axis(s, i, 1), v, rtol=1e-12, atol=0)
    assert np.array_equal(i, np.argsort(-s, axis=1, kind="stable")[:, :k])
    assert np.isfinite(v).all()


def test_item_factorised_scoring_matches_literal_under_permutation():
    rs = np.random.RandomState(3)
    nu, ni, H, k = 19, 26, 8, 5
    X = _binary(rs, nu, ni, 0.3)
    XT = X.T.copy()
    W1, b1, W2, b2 = _weights(rs, nu, H, nu)
    perm = rs.permutation(ni)
    assert (perm != np.arange(ni)).any()
    mask = X == 0
    v, i = autorec.get_recommendations_item(XT, W1, b1, W2, b2, perm, mask, k)
    Wt, V, b = autorec.item_operands(XT, W1, b1, W2, b2, perm)
    s = autorec.sigmoid(Wt @ V.T + b[:, None])                          # [U][I]: user u, column j = item perm[j]'s rows
    assert np.allclose(np.take_along_axis(np.where(mask, s, -np.inf), i, 1), v, rtol=1e-12, atol=0)
    # the same ranking on the logit (sigmoid is monotone; b2[u] is one offset per row)
    logit = np.where(mask, Wt @ V.T, -np.inf)
    assert np.array_equal(i, np.argsort(-logit, axis=1, kind="stable")[:, :k])
    # and NOT the unpermuted model's scores: column j is item perm[j]'s reconstruction
    v0, _ = autorec.get_recommendations_item(XT, W1, b1, W2, b2, np.arange(ni), mask, k)
    assert not np.allclose(v0, v)


def test_replay_matches_sparse_sampler_goldens():
    """samplers_tiny.npz holds two consecutive `random.sample(range(n), n)` draws after random.seed(42), as
    sparse_sampler.py makes them: UserAutoRec's two epochs, and ItemAutoRec's first epoch then first evaluation."""
    s = np.load(os.path.join(GOLD, "samplers_tiny.npz"))["vae_perm"]
    n = s.shape[1]
    state = random.getstate()
    user = autorec.replay(n, 99, 2, item=False)
    assert [k for k, _, _ in user] == ["epoch", "epoch"]
    assert [p for _, _, p in user] == s.tolist()
    item = autorec.replay(n, n, 2, item=True)
    assert [(k, e) for k, e, _ in item] == [("epoch", 0), ("eval", 0), ("epoch", 1), ("eval", 1)]
    assert item[0][2] == s[0].tolist() and item[1][2] == s[1].tolist()
    assert autorec.replay_restore(n) == s[0].tolist()
    skip = autorec.replay(n, n, 2, item=True, validation_rate=2)
    assert [(k, e) for k, e, _ in skip] == [("epoch", 0), ("epoch", 1), ("eval", 1)] and skip[1][2] == s[1].tolist()
    assert random.getstate() == state
