"""CPU checks of the CML restatements (oracle/cml.py): the literal B x B broadcast against an independent fp64 autodiff of
the same forward, and the O(B log B) counting form against the broadcast, ties at the margin and at -80 included."""
import numpy as np
import pytest
import torch

from oracle import cml


def _triples(rs, B, nu, ni):
    u = rs.randint(0, nu, B); i = rs.randint(0, ni, B); j = rs.randint(0, ni, B)
    u[: B // 3] = 0                                                     # duplicated users and items
    i[: B // 4] = 1; j[B // 5: B // 2] = 2
    return u, i, j


def _tables(rs, nu, ni, f, dyadic):
    """Rows and biases; dyadic=True: multiples of 1/8 and 1/64, so every fp64 sum is exact and pairs land exactly on
    the margin and on -80.  Items 3 and 4 sit near -80 and -90: their pairs fall below the clip."""
    if dyadic:
        Gu = rs.randint(-2, 3, (nu, f)) / 8.0; Gi = rs.randint(-2, 3, (ni, f)) / 8.0
        Bi = rs.randint(-32, 33, ni) / 64.0
        Bi[3], Bi[4] = -80.0, -90.0
    else:
        Gu = rs.uniform(-0.3, 0.3, (nu, f)); Gi = rs.uniform(-0.3, 0.3, (ni, f)); Bi = rs.uniform(-1, 1, ni)
        Bi[3], Bi[4] = -79.7, -90.3
    return Gu, Gi, Bi


def _with_clip_items(rs, i, j):
    k = rs.choice(len(i), size=max(1, len(i) // 8), replace=False)
    i, j = i.copy(), j.copy()
    i[k[::2]] = 3; i[k[1::2]] = 4
    return i, j


@pytest.mark.parametrize("B", [1, 7, 64])
def test_broadcast_backward_equals_autodiff(B):
    rs = np.random.RandomState(B)
    nu, ni, f = 9, 11, 5
    Gu, Gi, Bi = _tables(rs, nu, ni, f, dyadic=False)
    u, i, j = _triples(rs, B, nu, ni)
    i, j = _with_clip_items(rs, i, j)
    l_w, l_b, m = 0.01, 0.02, 0.5
    loss, dGu, dGi, dBi, n_a, n_b = cml.broadcast_step(Gu, Gi, Bi, u, i, j, l_w, l_b, m)
    tu, ti, tb = (torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in (Gu, Gi, Bi))
    gu, gp, gn = tu[u], ti[i], ti[j]
    bp, bn = tb[i], tb[j]
    xp = -((gu - gp) ** 2).sum(-1, keepdim=True) + bp
    xn = -((gu - gn) ** 2).sum(-1, keepdim=True) + bn
    diff = torch.clamp(xp - xn, -80.0, 1e8)                              # no pair sits on a bound: no tie conventions
    L = torch.clamp(m - diff, min=0).sum() + l_w * ((gu ** 2).sum() + (gp ** 2).sum() + (gn ** 2).sum()) / 2 \
        + l_b * (bp ** 2).sum() / 2 + l_b * (bn ** 2).sum() / 20
    L.backward()
    raw = (xp - xn).detach().numpy()
    assert np.abs(raw - m).min() > 1e-9 and np.abs(raw + 80).min() > 1e-9
    assert abs(loss - L.item()) <= 1e-12 * abs(L.item())
    for got, t in ((dGu, tu), (dGi, ti), (dBi, tb)):
        assert np.allclose(got, t.grad.numpy(), rtol=1e-12, atol=1e-12)
    if B > 1:
        assert (raw < -80).any() and 0 < n_a.sum() < B * B


@pytest.mark.parametrize("dyadic", [True, False], ids=["ties", "random"])
@pytest.mark.parametrize("B", [1, 2, 300, 4096])
def test_sorted_equals_broadcast(B, dyadic):
    rs = np.random.RandomState(B + dyadic)
    nu, ni, f = 40, 50, 6
    Gu, Gi, Bi = _tables(rs, nu, ni, f, dyadic)
    u, i, j = _triples(rs, B, nu, ni)
    i, j = _with_clip_items(rs, i, j)
    l_w, l_b, m = 0.01, 0.02, 0.5
    want = cml.broadcast_step(Gu, Gi, Bi, u, i, j, l_w, l_b, m)
    got = cml.sorted_step(Gu, Gi, Bi, u, i, j, l_w, l_b, m)
    assert np.array_equal(got[4], want[4]) and np.array_equal(got[5], want[5])
    tol = 0.0 if dyadic else 1e-12
    assert abs(got[0] - want[0]) <= tol * abs(want[0])
    for g, w in zip(got[1:4], want[1:4]):
        assert np.abs(g - w).max() <= tol * max(np.abs(w).max(), 1.0)
    if dyadic and B >= 300:                                             # the ties are there, on both sides of them
        D, E = cml.terms(Gu, Gi, Bi, u, i, j)
        x = D[:, None] + E[None, :]
        assert (x == m).sum() > 0 and (x == -80.0).sum() > 0 and (x < -80).sum() > 0


def test_count_le_edges():
    s = np.array([-1.0, 0.0, 0.0, 0.5, 2.0])
    assert cml.count_le([0.0, 0.5, -10.0, 10.0], s, 0.5).tolist() == [4, 3, 5, 0]
    assert cml.count_le([0.0], np.array([]), 0.5).tolist() == [0]
