"""CPU checks of oracle/dmf.py: the fp64 step against torch autograd (the batch-axis normalisation, Keras's clipped BCE,
columns below the 1e-12 floor), the factorised scoring against the literal get_recs restatement (short last block
included), and the host sampler restatement against the goldens the reference's own Sampler made."""
import os

import numpy as np
import pytest
import torch

from oracle import dmf

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _weights(rs, n_in, widths, scale):
    dims = [n_in] + list(widths)
    W = [rs.normal(0, scale, (n_in, dims[1]))] + [rs.normal(0, scale, (dims[l + 1], dims[l])) for l in range(1, len(widths))]
    b = [rs.normal(0, scale, w) for w in widths]
    return W, b


def _autograd(R, Wu, bu, Wi, bi, users, items, ratings, max_rating, cosine):
    t = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)
    P = [t(w) for w in Wu] + [t(x) for x in bu] + [t(w) for w in Wi] + [t(x) for x in bi]
    nu = len(Wu)

    def tower(X, W, b):
        h = X
        for l, w in enumerate(W):
            h = h @ (w if l == 0 else w.T) + b[l]
            if l < len(W) - 1:
                h = torch.relu(h)
        return h
    Rt = torch.tensor(R)
    U = tower(Rt[users], P[:nu], P[nu:2 * nu])
    V = tower(Rt.T[items], P[2 * nu:3 * nu], P[3 * nu:])
    if cosine:                               # tf.nn.l2_normalize(x, 0) = x * rsqrt(maximum(sum x^2, eps))
        U = U * torch.rsqrt(torch.maximum((U * U).sum(0, keepdim=True), torch.tensor(1e-12, dtype=torch.float64)))
        V = V * torch.rsqrt(torch.maximum((V * V).sum(0, keepdim=True), torch.tensor(1e-12, dtype=torch.float64)))
    o = (U * V).sum(1)
    y = torch.tensor(ratings, dtype=torch.float64) / max_rating
    p = torch.clamp(o, dmf.BCE_EPS, dmf.BCE_HI)           # float32 bounds, as Keras computes them
    loss = -(y * torch.log(p + dmf.BCE_EPS) + (1 - y) * torch.log(1 - p + dmf.BCE_EPS)).mean()
    loss.backward()
    return loss.item(), [x.grad.numpy() for x in P], o.detach().numpy()


def _data(rs, nu, ni, density=0.3):
    R = np.where(rs.rand(nu, ni) < density, rs.randint(1, 6, (nu, ni)), 0).astype(np.float64)
    R[:, 0] = np.where(R[:, 0] == 0, 3, R[:, 0])
    return R


@pytest.mark.parametrize("cosine", [True, False])
@pytest.mark.parametrize("B,widths", [(1, (8,)), (7, (16, 8)), (64, (32, 16, 8)), (300, (64, 32))])
def test_step_matches_autograd(cosine, B, widths):
    rs = np.random.RandomState(B + len(widths))
    nu, ni = 30, 40
    R = _data(rs, nu, ni)
    scale = 0.3 if cosine else 0.05
    Wu, bu = _weights(rs, ni, widths, scale)
    Wi, bi = _weights(rs, nu, widths, scale)
    users = rs.randint(0, nu, B); items = rs.randint(0, ni, B)
    users[: B // 3] = 2; items[B // 4: B // 2] = 5                     # repeated users and items
    ratings = np.where(rs.rand(B) < 0.3, R[users, items], 0.0)
    got = dmf.step(R, Wu, bu, Wi, bi, users, items, ratings, 5.0, cosine)
    loss, grads, o = _autograd(R, Wu, bu, Wi, bi, users, items, ratings, 5.0, cosine)
    assert got[0] == pytest.approx(loss, rel=1e-12)
    assert np.allclose(got[5], o, rtol=1e-12, atol=1e-15)
    mine = got[1] + got[2] + got[3] + got[4]
    for a, b in zip(mine, grads):
        assert np.allclose(a, b, rtol=1e-10, atol=1e-14)


def test_step_clipped_outputs_and_floored_columns():
    """Outputs below 1e-7 pass no gradient, and a column whose batch sum of squares is below 1e-12 gets only
    the direct term (Maximum's gradient goes to the floor)."""
    rs = np.random.RandomState(3)
    nu, ni, B = 20, 25, 40
    R = _data(rs, nu, ni, 0.5)
    Wu, bu = _weights(rs, ni, (16, 8), 0.5)
    Wi, bi = _weights(rs, nu, (16, 8), 0.5)
    for W, b in ((Wu, bu), (Wi, bi)):                                 # column 0 of both outputs ~1e-8 per row
        W[-1][0] *= 1e-9; b[-1][0] = 1e-8
    users = rs.randint(0, nu, B); items = rs.randint(0, ni, B)
    ratings = R[users, items]
    got = dmf.step(R, Wu, bu, Wi, bi, users, items, ratings, 5.0, True)
    U = got[6]
    assert (U[:, 0] ** 2).sum() < 1e-12
    o = got[5]
    assert (o < dmf.BCE_EPS).any() and ((o >= dmf.BCE_EPS) & (o <= dmf.BCE_HI)).any()
    loss, grads, _ = _autograd(R, Wu, bu, Wi, bi, users, items, ratings, 5.0, True)
    assert got[0] == pytest.approx(loss, rel=1e-12)
    for a, b in zip(got[1] + got[2] + got[3] + got[4], grads):
        assert np.allclose(a, b, rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize("cosine", [True, False])
@pytest.mark.parametrize("block", [4, 7, 50])
def test_factorised_scoring_matches_literal_get_recs(cosine, block):
    rs = np.random.RandomState(block)
    nu, ni = 17, 9
    R = _data(rs, nu, ni)
    Wu, bu = _weights(rs, ni, (16, 8), 0.3)
    Wi, bi = _weights(rs, nu, (16, 8), 0.3)
    Wi[-1][3] *= 1e-9; bi[-1][3] = 0.0                                  # tiny item factors: B V^2 below the floor
    Uo = dmf.tower(R, Wu, bu)[0]
    Vo = dmf.tower(R.T, Wi, bi)[0]
    Uh, Vh = dmf.score_operands(Uo, Vo, block, cosine)
    bl = min(block, nu)
    for o in range(0, nu, bl):
        e = min(o + bl, nu)
        want = dmf.get_recs_literal(R, Wu, bu, Wi, bi, o, e, cosine)
        got = Uh[o:e] @ Vh[e - o].T
        assert np.allclose(got, want, rtol=1e-12, atol=1e-15), (o, e)
    if cosine and nu % bl:
        assert len(Vh) == 2                                              # the short last block has its own item operand


def test_host_sampler_matches_goldens():
    g = np.load(os.path.join(GOLD, "dmf_sampler_cases.npz"))
    for name in g["names"]:
        n_users, n_items, neg, events, _ = (int(x) for x in g[f"{name}_meta"])
        p, rows, rat = g[f"{name}_indptr"], g[f"{name}_rows"], g[f"{name}_ratings"]
        s = dmf.Sampler([rows[p[u]:p[u + 1]].tolist() for u in range(n_users)],
                        [rat[p[u]:p[u + 1]].tolist() for u in range(n_users)], n_items, neg)
        for e in range(2):
            u, i, r = s.epoch(events)
            assert np.array_equal(u, g[f"{name}_e{e}_u"]), (name, e)
            assert np.array_equal(i, g[f"{name}_e{e}_i"]), (name, e)
            assert np.array_equal(r, g[f"{name}_e{e}_r"]), (name, e)
        if neg == 0:
            assert (g[f"{name}_e0_r"] > 0).all()
