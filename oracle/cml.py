"""fp64 NumPy restatements of the reference's CML (latent_factor_models/CML/CML_model.py).  TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED, as for every TensorFlow model here (oracle/tf_models.py): tensorflow==2.3.2 is absent, so these follow
the model code line by line plus the TF 2.3 semantics it relies on:
  - the sampler's (B, 1) index arrays: `tf.squeeze(Bi(item))` is (B,), the row gathers squeeze to (B, f) (f >= 2), and
    `reduce_sum(..., keepdims=True)` is (B, 1), so `-l2 + beta` broadcasts to B x B (CML_model.py:59-72);
  - tf.nn.l2_loss(t) = sum(t**2)/2; clip_by_value passes the gradient only strictly inside (-80, 1e8) (the convention
    oracle/tf_models.py states for BPRMF_batch); Maximum passes it to its first argument on ties (x >= y);
  - gradients w.r.t. the tables are IndexedSlices whose duplicate indices are summed; Keras Adam is tf_models.KerasAdam.
`m` is the margin as the fp32 constant TF makes of it, widened.

Two restatements of the loss and gradients: `broadcast_step`, the literal B x B forward and its backward (B up to a few
thousand), and `sorted_step`, the O(B log B) counting form the device uses (csrc/cml.cu): with D_a = q_a - p_a and
E_b = Bi[pos_b] - Bi[neg_b], pair (a, b) is active when -80 < D_a + E_b <= m, n_a / n'_b count a's / b's active pairs, and
    hinge = sum_a [(m + 80) #{b : D_a + E_b <= -80} + (m - D_a) n_a] - sum_b n'_b E_b.
tests/test_oracle_cml.py checks the first against an independent autodiff and the second against the first."""
import numpy as np

CLIP_LO, CLIP_HI = -80.0, 1e8


def broadcast_step(Gu, Gi, Bi, u, i, j, l_w, l_b, m):
    """CML_model.call/train_step (:59-98) on fp64 tables (Gu [n_users, f], Gi [n_items, f], Bi [n_items]) for the triples
    (u, i, j): (loss, dGu, dGi, dBi, n_a, n'_b), the B x B difference formed as the reference forms it."""
    beta_pos, gamma_u, gamma_pos = Bi[i], Gu[u], Gi[i]
    beta_neg, gamma_neg = Bi[j], Gi[j]
    l2_pos = ((gamma_u - gamma_pos) ** 2).sum(-1, keepdims=True)              # (B, 1)
    l2_neg = ((gamma_u - gamma_neg) ** 2).sum(-1, keepdims=True)
    xu_pos = -l2_pos + beta_pos                                               # (B, B): row a, column b
    xu_neg = -l2_neg + beta_neg
    raw = xu_pos - xu_neg
    difference = np.clip(raw, CLIP_LO, CLIP_HI)
    loss = np.maximum(m - difference, 0).sum()
    loss += l_w * ((gamma_u ** 2).sum() + (gamma_pos ** 2).sum() + (gamma_neg ** 2).sum()) / 2 \
        + l_b * (beta_pos ** 2).sum() / 2 + l_b * (beta_neg ** 2).sum() / 2 / 10
    active = (m - difference >= 0) & (raw > CLIP_LO) & (raw < CLIP_HI)       # d loss / d raw = -1 there, else 0
    n_a, n_b = active.sum(1), active.sum(0)
    # d loss / d l2_pos[a] = +n_a, d loss / d l2_neg[a] = -n_a, d loss / d beta_pos[b] = -n'_b, d loss / d beta_neg[b] = +n'_b
    dGu = np.zeros_like(Gu); dGi = np.zeros_like(Gi); dBi = np.zeros_like(Bi)
    na = n_a[:, None].astype(np.float64)
    np.add.at(dGu, u, 2 * na * (gamma_u - gamma_pos) - 2 * na * (gamma_u - gamma_neg) + l_w * gamma_u)
    np.add.at(dGi, i, -2 * na * (gamma_u - gamma_pos) + l_w * gamma_pos)
    np.add.at(dGi, j, 2 * na * (gamma_u - gamma_neg) + l_w * gamma_neg)
    np.add.at(dBi, i, -n_b + l_b * beta_pos)
    np.add.at(dBi, j, n_b + l_b * beta_neg / 10)
    return loss, dGu, dGi, dBi, n_a, n_b


def count_le(x, s, t):
    """#{k : x + s[k] <= t} for every x, s sorted ascending, the sum in fp64: binary lifting on the prefix where the
    predicate holds, as csrc/cml.cu counts."""
    x = np.asarray(x, np.float64); s = np.asarray(s, np.float64)
    n = len(s)
    c = np.zeros(len(x), np.int64)
    step = 1
    while step * 2 <= n:
        step *= 2
    while n > 0 and step > 0:
        k = c + step
        ok = k <= n
        ok[ok] = x[ok] + s[k[ok] - 1] <= t
        c = np.where(ok, k, c)
        step //= 2
    return c


def terms(Gu, Gi, Bi, u, i, j):
    """(D, E) in fp64"""
    gu = Gu[u]
    return ((gu - Gi[j]) ** 2).sum(1) - ((gu - Gi[i]) ** 2).sum(1), Bi[i] - Bi[j]


def sorted_step(Gu, Gi, Bi, u, i, j, l_w, l_b, m, D=None, E=None):
    """The same loss and gradients as broadcast_step in O(B log B) (searchsorted-style counting); D, E default to
    terms(...), and may be given (e.g. a kernel's fp32 terms) to classify the pairs on exactly those values."""
    if D is None:
        D, E = terms(Gu, Gi, Bi, u, i, j)
    D = np.asarray(D, np.float64); E = np.asarray(E, np.float64)
    Ds, Es = np.sort(D), np.sort(E)
    below_a = count_le(D, Es, CLIP_LO)
    n_a = count_le(D, Es, m) - below_a
    n_b = count_le(E, Ds, m) - count_le(E, Ds, CLIP_LO)
    gu, gp, gn, bp, bn = Gu[u], Gi[i], Gi[j], Bi[i], Bi[j]
    loss = ((m - CLIP_LO) * below_a + (m - D) * n_a).sum() - (n_b * E).sum()
    loss += l_w * ((gu ** 2).sum() + (gp ** 2).sum() + (gn ** 2).sum()) / 2 + l_b * (bp ** 2).sum() / 2 \
        + l_b * (bn ** 2).sum() / 20
    na = 2.0 * n_a[:, None]
    dGu = np.zeros_like(Gu); dGi = np.zeros_like(Gi); dBi = np.zeros_like(Bi)
    np.add.at(dGu, u, -na * (gp - gn) + l_w * gu)
    np.add.at(dGi, i, -na * (gu - gp) + l_w * gp)
    np.add.at(dGi, j, na * (gu - gn) + l_w * gn)
    np.add.at(dBi, i, -n_b + l_b * bp)
    np.add.at(dBi, j, n_b + l_b * bn / 10)
    return loss, dGu, dGi, dBi, n_a, n_b


def predict(Gu, Gi, Bi, start, stop):
    """CML_model.predict (:101-106): -sum((Gu[start:stop, None] - Gi)^2, -1) + Bi, fp64."""
    return -(((Gu[start:stop, None, :] - Gi[None, :, :]) ** 2).sum(-1)) + Bi[None, :]


def expansion_bound(Gu, Gi, Bi, users, unit):
    """Per user, a bound on |fp32 list value - predict| when the scorer ranks (2 Gu, Gi, c = Bi - |Gi|^2) and -|Gu|^2 is
    added to the kept values, every operand rounded to `unit`:
      - the scorer, by oracle/topk_bound.py's rule with c as the bias: (d + 2) unit (2 |gu| vmax + cmax);
      - c and |gu|^2, each a d-term fp32 sum of squares and one addition: (d + 2) unit (vmax^2 + bmax) and
        (d + 2) unit |gu|^2;
      - the final addition: unit times the value, at most unit ((|gu| + vmax)^2 + bmax).
    With cmax <= vmax^2 + bmax, the sum is at most (d + 3) unit ((|gu| + vmax)^2 + 2 vmax^2 + 2 bmax)."""
    d = Gu.shape[1]
    nu = np.sqrt((Gu[users] ** 2).sum(1))
    vmax = np.sqrt((Gi ** 2).sum(1)).max()
    bmax = np.abs(Bi).max()
    return (d + 3) * unit * ((nu + vmax) ** 2 + 2 * vmax ** 2 + 2 * bmax)
