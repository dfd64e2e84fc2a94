"""CPU checks of oracle/convneumf.py, the fp64 restatement the ConvNeuMF GPU tests compare against: the literal
map-and-conv forward against torch.nn.functional.conv2d on the [B, 1, f, f] map and against the quad-tree form, the
hand-written backward against torch.autograd, the coordinates the network never reads, the GlorotUniform limits and
one Keras Adam step."""
import numpy as np
import pytest
import torch

from oracle import convneumf as oracle

GEOMS = [(8, [8]), (8, [8, 16]), (8, [8, 16, 8]), (100, [16]), (100, [16, 32]), (100, [8, 16, 24]), (101, [8]),
         (101, [16, 8]), (101, [8, 8, 16])]


def _torch_forward(P, U, I, tu, ti, masks=None):
    """The reference's call() in torch fp64: conv2d on the [B, 1, f, f] map (NCHW), relu, spatial sum, the head."""
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    x = (U[tu][:, :, None] * I[ti][:, None, :])[:, None]
    ks = [(P["W1"], P["b1"])] + [(P["K"][l], P["b"][l]) for l in range(2, len(P["K"]))]
    for K, b in ks:
        x = torch.relu(torch.nn.functional.conv2d(x, K.permute(3, 2, 0, 1), b, stride=2))
    s = x.sum(dim=(2, 3))
    m1, m2 = (None, None) if masks is None else masks
    x1 = s if m1 is None else s * t(m1)
    z = x1 @ P["Wd1"] + P["bd1"]
    x2 = z if m2 is None else z * t(m2)
    return x2 @ P["wd2"] + P["bd2"][0]


def _tparams(P):
    tp = {}
    for k, v in P.items():
        if isinstance(v, list):
            tp[k] = [None if a is None else torch.tensor(a, requires_grad=True) for a in v]
        else:
            tp[k] = torch.tensor(v, requires_grad=True)
    return tp


@pytest.mark.parametrize("f,widths", GEOMS)
def test_literal_forward_matches_conv2d_and_quadtree(f, widths):
    rs = np.random.default_rng(f + len(widths))
    P = oracle.init_params(rs, widths)
    U, I = rs.normal(0, 1, (6, f)), rs.normal(0, 1, (7, f))
    tu, ti = np.array([0, 1, 1, 5, 0]), np.array([2, 2, 3, 6, 2])        # repeated users and items
    y_lit, last = oracle.literal_forward(P, U[tu], I[ti])
    y_qt, h, _ = oracle.quadtree_forward(P, U[tu], I[ti])
    with torch.no_grad():
        y_t = _torch_forward(_tparams(P), torch.tensor(U), torch.tensor(I), tu, ti).numpy()
    scale = np.abs(y_t).max() + 1
    assert np.abs(y_lit - y_t).max() <= 1e-12 * scale
    assert np.abs(y_qt - y_t).max() <= 1e-12 * scale
    HL, _ = oracle.geometry(f, len(widths))
    assert last.shape[1:3] == (HL, HL) and h[len(widths)].shape[1] == HL * HL


@pytest.mark.parametrize("f,widths", GEOMS)
@pytest.mark.parametrize("dropout", [False, True])
def test_gradients_match_autograd(f, widths, dropout):
    rs = np.random.default_rng(3 * f + len(widths))
    P = oracle.init_params(rs, widths)
    nu, ni, B = 5, 6, 9
    U, I = rs.uniform(-1, 1, (nu, f)), rs.uniform(-1, 1, (ni, f))
    tu = np.array([0, 0, 1, 2, 3, 4, 0, 1, 1]); ti = rs.integers(0, ni, B); tj = rs.integers(0, ni, B)
    ti[:3] = ti[0]
    cL, l_w = widths[-1], 0.01
    masks = None
    if dropout:
        keep = lambda: (rs.random((B, cL)) > 0.25) / 0.75
        masks = (keep(), keep(), keep(), keep())
    loss, G, dU, dI, _ = oracle.loss_and_grads(P, U, I, tu, ti, tj, l_w, masks)
    tp = _tparams(P)
    Ut, It = torch.tensor(U, requires_grad=True), torch.tensor(I, requires_grad=True)
    yp = _torch_forward(tp, Ut, It, tu, ti, None if masks is None else masks[:2])
    yn = _torch_forward(tp, Ut, It, tu, tj, None if masks is None else masks[2:])
    x = torch.clamp(yp - yn, -80, 1e8)
    tl = torch.nn.functional.softplus(-x).sum() + l_w * ((Ut[tu] ** 2).sum() + (It[ti] ** 2).sum() + (It[tj] ** 2).sum()) / 2
    tl.backward()
    assert loss == pytest.approx(tl.item(), rel=1e-10)
    pairs = [(G["W1"], tp["W1"]), (G["b1"], tp["b1"]), (G["Wd1"], tp["Wd1"]), (G["bd1"], tp["bd1"]), (G["wd2"], tp["wd2"]),
             (G["bd2"], tp["bd2"]), (dU, Ut), (dI, It)]
    pairs += [(G["K"][l], tp["K"][l]) for l in range(2, len(widths) + 1)]
    pairs += [(G["b"][l], tp["b"][l]) for l in range(2, len(widths) + 1)]
    for mine, ref in pairs:
        r = ref.grad.numpy()
        assert np.abs(mine - r).max() <= 1e-8 * (np.abs(r).max() + 1), ref.shape


def test_coordinates_beyond_m_get_only_the_regulariser():
    f, widths = 101, [8, 16]                                            # m = 100
    rs = np.random.default_rng(0)
    P = oracle.init_params(rs, widths)
    U, I = rs.uniform(-1, 1, (4, f)), rs.uniform(-1, 1, (5, f))
    tu, ti, tj = np.array([0, 0, 3]), np.array([1, 2, 1]), np.array([4, 4, 0])
    _, _, dU, dI, _ = oracle.loss_and_grads(P, U, I, tu, ti, tj, 0.02)
    cu = np.bincount(tu, minlength=4); ci = np.bincount(np.concatenate([ti, tj]), minlength=5)
    assert np.allclose(dU[:, 100], 0.02 * cu * U[:, 100]) and np.allclose(dI[:, 100], 0.02 * ci * I[:, 100])
    # and the scores do not depend on them
    y0 = oracle.full_scores(P, U, I)
    U2, I2 = U.copy(), I.copy(); U2[:, 100] = 7.0; I2[:, 100] = -3.0
    assert np.array_equal(oracle.full_scores(P, U2, I2), y0)


def test_glorot_limits_use_conv_fans():
    lim = oracle.glorot_limits([32, 32])
    assert lim["W1"] == pytest.approx(np.sqrt(6 / (4 * 1 + 4 * 32)))
    assert lim["K2"] == pytest.approx(np.sqrt(6 / (4 * 32 + 4 * 32)))
    assert lim["Wd1"] == pytest.approx(np.sqrt(6 / 64)) and lim["wd2"] == pytest.approx(np.sqrt(6 / 33))
    P = oracle.init_params(np.random.default_rng(1), [32, 32])
    assert np.abs(P["W1"]).max() <= lim["W1"] and np.abs(P["K"][2]).max() <= lim["K2"]


def test_adam_step_is_keras_adam():
    rs = np.random.default_rng(2)
    P = oracle.init_params(rs, [8])
    U, I = rs.uniform(-1, 1, (3, 8)), rs.uniform(-1, 1, (4, 8))
    loss, G, dU, dI, _ = oracle.loss_and_grads(P, U, I, np.array([0, 1]), np.array([1, 2]), np.array([3, 0]), 0.005)
    W0, U0 = P["W1"].copy(), U.copy()
    opt = oracle.KerasAdam(1e-3)
    oracle.adam_step(opt, P, U, I, G, dU, dI)
    lr_t = 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9)
    g = G["W1"]
    want = W0 - lr_t * (0.1 * g) / (np.sqrt(0.001 * g * g) + 1e-7)
    assert np.allclose(P["W1"], want, rtol=1e-12, atol=1e-15)
    gu = dU
    assert np.allclose(U, U0 - lr_t * (0.1 * gu) / (np.sqrt(0.001 * gu * gu) + 1e-7), rtol=1e-12, atol=1e-15)
