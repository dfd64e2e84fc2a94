"""CPU checks of oracle/pointwise_mf.py: the MF / PMF / FM / LMF restatements against fp64 torch autograd of the
reference's forward formulas (LMF's g_u regulariser included: it is in the loss and has no gradient on the item side),
TF's sparse Adagrad on the touched rows against the dense pass, the LMF epoch, and the rating-label pass on a hand-made
CSR."""
import numpy as np
import pytest
import torch

from oracle import pointwise_mf as pm


def _tables(rs, nu, ni, f, biases):
    T = {"P": rs.randn(nu, f) * 0.5, "Q": rs.randn(ni, f) * 0.5}
    if biases:
        T["bu"], T["bi"], T["g"] = rs.randn(nu) * 0.3, rs.randn(ni) * 0.3, 0.17
    return T


def _batch(rs, nu, ni, B):
    u = rs.randint(0, nu, B); u[:5] = 0                                   # repeated users and items
    i = rs.randint(0, ni, B); i[3:9] = 1
    return u, i


@pytest.mark.parametrize("model", ["MF", "PMF", "FM"])
def test_mse_models_against_autograd(model):
    rs = np.random.RandomState(1)
    nu, ni, f, B = 13, 17, 6, 40
    T = _tables(rs, nu, ni, f, model == "FM")
    u, i = _batch(rs, nu, ni, B)
    y = rs.randint(0, 6, B).astype(np.float64) if model == "FM" else rs.randint(0, 2, B).astype(np.float64)
    fn = {"MF": pm.mf_forward_backward, "PMF": pm.pmf_forward_backward, "FM": pm.fm_forward_backward}[model]
    loss, G, out = fn(T, u, i, y)
    t = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in T.items()}
    x = (t["P"][u] * t["Q"][i]).sum(1)
    if model == "FM":
        x = x + t["g"] + t["bu"][u] + t["bi"][i]
    if model == "PMF":
        x = torch.sigmoid(x)
    ref = ((x - torch.tensor(y)) ** 2).mean()
    ref.backward()
    assert abs(loss - ref.item()) < 1e-13 and np.allclose(out, x.detach().numpy(), rtol=1e-14, atol=1e-14)
    for k in T:
        assert np.allclose(G[k], t[k].grad.numpy(), rtol=1e-12, atol=1e-14), k


def test_lmf_item_side_against_autograd_with_user_regulariser():
    rs = np.random.RandomState(2)
    nu, ni, f, B, alpha, reg = 11, 19, 5, 50, 0.5, 0.1
    T = {"Gu": rs.randn(nu, f), "Gi": rs.randn(ni, f), "Bu": rs.randn(nu) * 0.2, "Bi": rs.randn(ni) * 0.2}
    u, i = _batch(rs, nu, ni, B)
    y = rs.randint(0, 2, B).astype(np.float64)
    T["Gu"][0] *= 60                                                        # |x| > 90: the literal log(1 + e^x) overflows fp32
    loss, G, x = pm.lmf_forward_backward(T, u, i, y, alpha, reg)
    assert np.abs(x).max() > 90 and np.isfinite(loss)
    t = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in T.items()}
    xt = (t["Gu"][u] * t["Gi"][i]).sum(1) + t["Bu"][u] + t["Bi"][i]
    ay = alpha * torch.tensor(y)
    ref = (-(ay * xt - (1 + ay) * torch.nn.functional.softplus(xt))).sum() \
        + reg * ((t["Gu"][u] ** 2).sum() / 2 + (t["Gi"][i] ** 2).sum() / 2)
    ref.backward()
    assert abs(loss - ref.item()) <= 1e-12 * abs(ref.item())
    assert set(G) == {"Gi", "Bi"}                                            # the item branch differentiates Gi, Bi only
    for k in G:
        assert np.allclose(G[k], t[k].grad.numpy(), rtol=1e-12, atol=1e-12), k
    # the g_u term is in the loss: it is the loss at reg = 0 plus reg / 2 (sum |g_u|^2 + sum |g_i|^2) over the batch rows
    l0, _, _ = pm.lmf_forward_backward(T, u, i, y, alpha, 0.0)
    gu2 = (T["Gu"][u] ** 2).sum()
    assert gu2 > 0 and abs(loss - (l0 + reg * (gu2 + (T["Gi"][i] ** 2).sum()) / 2)) <= 1e-12 * abs(loss)


def test_touched_row_adagrad_equals_dense():
    rs = np.random.RandomState(3)
    n, f = 30, 7
    var, acc = rs.randn(n, f), np.full((n, f), pm.ADAGRAD_INIT)
    rows = np.array([4, 9, 4, 4, 17, 9, 0])
    row_grads = rs.randn(len(rows), f)
    dense = np.zeros((n, f)); np.add.at(dense, rows, row_grads)
    v1, a1, v2, a2 = var.copy(), acc.copy(), var.copy(), acc.copy()
    pm.adagrad_sparse(v1, a1, rows, row_grads, 0.05)
    pm.adagrad_dense(v2, a2, dense, 0.05)
    assert np.array_equal(v1, v2) and np.array_equal(a1, a2)
    untouched = np.setdiff1d(np.arange(n), rows)
    assert np.array_equal(v1[untouched], var[untouched]) and np.array_equal(a1[untouched], acc[untouched])


def test_lmf_epoch_is_two_item_passes_on_one_stream():
    rs = np.random.RandomState(4)
    nu, ni, f, Ts, B = 9, 14, 4, 37, 8
    T = {"Gu": rs.randn(nu, f) * 0.3, "Gi": rs.randn(ni, f) * 0.3, "Bu": np.zeros(nu), "Bi": np.zeros(ni)}
    acc = {"Gi": np.full((ni, f), pm.ADAGRAD_INIT), "Bi": np.full(ni, pm.ADAGRAD_INIT)}
    stream = (rs.randint(0, nu, 2 * Ts), rs.randint(0, ni, 2 * Ts), rs.randint(0, 2, 2 * Ts).astype(np.float64))
    Gu0, Bu0 = T["Gu"].copy(), T["Bu"].copy()
    W = {k: v.copy() for k, v in T.items()}; A = {k: v.copy() for k, v in acc.items()}
    total = pm.lmf_epoch(T, acc, stream, Ts, B, 0.5, 0.1, 0.05)
    want = 0.0                                                              # step by step: 5 + 5 batches, the last ones short
    for lo, hi in [(s, min(s + B, Ts)) for s in range(0, Ts, B)] + [(s, min(s + B, 2 * Ts)) for s in range(Ts, 2 * Ts, B)]:
        loss, G, _ = pm.lmf_forward_backward(W, stream[0][lo:hi], stream[1][lo:hi], stream[2][lo:hi], 0.5, 0.1)
        want += loss
        for k in G:
            pm.adagrad_dense(W[k], A[k], G[k], 0.05)
    assert total == want and all(np.array_equal(T[k], W[k]) for k in T)
    assert np.array_equal(T["Gu"], Gu0) and np.array_equal(T["Bu"], Bu0)


def test_rating_labels_on_hand_made_csr():
    indptr = np.array([0, 3, 3, 5])
    indices = np.array([1, 4, 7, 0, 2])                                     # sorted rows: {1, 4, 7}, {}, {0, 2}
    ratings = np.array([5.0, 3.0, 1.0, 4.0, 2.0])
    u = np.array([0, 0, 0, 2, 2, 1, 0])
    i = np.array([7, 1, 3, 2, 1, 5, 4])
    y = np.array([1, 1, 0, 1, 0, 0, 1])
    assert np.array_equal(pm.rating_labels(indptr, indices, ratings, u, i, y), [1.0, 5.0, 0.0, 2.0, 0.0, 0.0, 3.0])
    with pytest.raises(AssertionError):
        pm.rating_labels(indptr, indices, ratings, np.array([0]), np.array([3]), np.array([1]))


def test_full_scores():
    rs = np.random.RandomState(5)
    T = _tables(rs, 4, 6, 3, True)
    s = T["P"] @ T["Q"].T
    assert np.array_equal(pm.full_scores("MF", T), s)
    assert np.allclose(pm.full_scores("PMF", T), 1 / (1 + np.exp(-s)), rtol=1e-15)
    assert np.allclose(pm.full_scores("FM", T), s + T["bu"][:, None] + T["bi"] + T["g"], rtol=1e-15)
    L = {"Gu": T["P"], "Gi": T["Q"], "Bu": T["bu"], "Bi": T["bi"]}
    assert np.allclose(pm.full_scores("LMF", L), s + T["bu"][:, None] + T["bi"], rtol=1e-15)
