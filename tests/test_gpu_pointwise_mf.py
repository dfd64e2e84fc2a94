"""GPU tests of MF, PMF, FM and LMF (csrc/pointwise_mf.cu, the null-bias form of eb_rating_mf_step_f32,
recommender/rating_mf.py, recommender/logistic_mf.py): the step kernels against the fp64 restatements of
oracle/pointwise_mf.py at bounds derived from f and the fp32 unit roundoff, the touched-row Adagrad, the rating-label
pass, one Adam step, the top-k against the fp64 bound of oracle/topk_bound.py, the rank and pair passes, C1 runs through
run_experiment, and the refusals.

Bounds (u = 2^-24, gamma(n) = n u / (1 - n u)): a dot of n fp32 products is within gamma(n) sum |p_k q_k| of the exact
value; expf / log1pf / sqrtf and the IEEE division are within 2 ulp, so sigmoid and softplus add at most 8 u relative.  An
error dx in the logit moves PMF's e = 2 (o - y) o (1 - o) / B by at most dx * 2 / B (|de/dx| <= 2 / B since |o - y| <= 1
and |d(o (1 - o))/dx| <= 1/4, |o (1 - o)| <= 1/4) and LMF's c = sigmoid(x)(1 + a y) - a y by dx (1 + a y) / 4.  An atomic
sum of m contributions in any order is within gamma(m) of their absolute sum.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import yaml

from elliot_b200 import ops, synth_c1
from oracle import pointwise_mf as pm
from oracle import tf_models as tfm
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 2.0 ** -24
gam = lambda n: n * U32 / (1 - n * U32)
CONFIG = {"MF": {"bias": "none"}, "PMF": {"bias": "none", "init": "normal", "head": "sigmoid"},
          "FM": {"bias": "zero", "global_bias": True}}
d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _csr(nu, ni, seed):
    rs = np.random.RandomState(seed)
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, min(40, ni - 1)), replace=False)) for _ in range(nu)]
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


def _model(name, nu, ni, f, indptr, indices, seed=3):
    from elliot_b200.recommender.logistic_mf import LMFModel
    from elliot_b200.recommender.rating_mf import RatingMFModel
    if name == "LMF":
        m = LMFModel(nu, ni, f, 0.1, 0.5, 0.05, seed, DEV)
        m.P["Bu"].normal_(0, 0.3); m.P["Bi"].normal_(0, 0.3)
        return m
    m = RatingMFModel(nu, ni, f, 1e-3, seed, d(indptr), d(indices), False, DEV, **CONFIG[name])
    if name == "FM":
        m.P["bu"][:nu].normal_(0, 0.2); m.P["bi"][:ni].normal_(0, 0.2); m.P["g"][0] = 0.31
    if name == "PMF":                                                   # logits of order 1, so the sigmoid's slope matters
        m.P["P"][:, :f] *= 40; m.P["Q"][:, :f] *= 40
    return m


def _host(m, name, f):
    if name == "LMF":
        return {"Gu": m.P["Gu"][:, :f].double().cpu().numpy(), "Gi": m.P["Gi"][:, :f].double().cpu().numpy(),
                "Bu": m.P["Bu"].double().cpu().numpy(), "Bi": m.P["Bi"].double().cpu().numpy()}
    T = {"P": m.P["P"][:, :f].double().cpu().numpy(), "Q": m.P["Q"][:, :f].double().cpu().numpy()}
    if "bu" in m.P:
        T["bu"] = m.P["bu"][:m.nu].double().cpu().numpy(); T["bi"] = m.P["bi"][:m.ni].double().cpu().numpy()
    if "g" in m.P:
        T["g"] = float(m.P["g"][0])
    return T


def _batch(rs, nu, ni, B, name):
    u = rs.randint(0, nu, B).astype(np.int32); it = rs.randint(0, ni, B).astype(np.int32)
    if B > 8:
        u[:B // 8] = 1; it[B // 16:B // 8 + 3] = 2                      # repeated users and items
    y = (rs.randint(0, 6, B) if name == "FM" else rs.randint(0, 2, B)).astype(np.float32)
    return u, it, y


def _scatter_abs(n, idx, rows):
    out = np.zeros((n,) + rows.shape[1:]); np.add.at(out, idx, np.abs(rows)); return out


def _check_mse_step(m, name, f, u, it, y):
    """The step (null-bias MF, PMF, FM) against the fp64 restatement, every element within its derived bound."""
    T = _host(m, name, f)
    fn = {"MF": pm.mf_forward_backward, "PMF": pm.pmf_forward_backward, "FM": pm.fm_forward_backward}[name]
    u64 = u.astype(np.int64)
    loss_ref, G, out = fn(T, u64, it, y.astype(np.float64))
    B = len(u)
    S = np.abs(T["P"][u64] * T["Q"][it]).sum(1)                          # sum |p_k q_k| per sample
    if name == "FM":
        S = S + np.abs(T["bu"][u64]) + np.abs(T["bi"][it]) + abs(T["g"])
    dx = gam(f + 4) * S + U32 * np.abs(y)                                # the error of out - y before the head
    if name == "PMF":
        de = 2.0 / B * dx + 16 * U32 * np.abs(2 * (out - y) * out * (1 - out) / B)
        e = 2 * (out - y) * out * (1 - out) / B
    else:
        de = 2.0 / B * dx + 2 * U32 * np.abs(2 * (out - y) / B)
        e = 2 * (out - y) / B
    m._loss.zero_()
    m.grads((d(u), d(it), d(y)))
    torch.cuda.synchronize()
    dd = out - y
    dd_err = (dx / 4 + 8 * U32) if name == "PMF" else dx
    assert abs(m._loss.item() - loss_ref) <= ((2 * np.abs(dd) * dd_err + dd_err ** 2).sum() + 4 * U32 * (dd * dd).sum()) / B + 1e-300
    mult = max(np.bincount(u).max(), np.bincount(it).max())
    for k, (rows, other) in {"Q": (it, T["P"][u64]), "P": (u64, T["Q"][it])}.items():
        n = T[k].shape[0]
        bound = _scatter_abs(n, rows, other * de[:, None]) + (U32 + gam(mult)) * _scatter_abs(n, rows, other * e[:, None]) * 2
        got = m.G[k][:, :f].double().cpu().numpy()
        assert (np.abs(got - G[k]) <= bound + 1e-30).all(), k
        assert not m.G[k][:, f:].any()
    if name == "FM":
        for k, rows in (("bu", u64), ("bi", it)):
            n = T[k].shape[0]
            bound = _scatter_abs(n, rows, de) + (U32 + gam(mult)) * _scatter_abs(n, rows, e) * 2
            assert (np.abs(m.G[k][:n].double().cpu().numpy() - G[k]) <= bound + 1e-30).all(), k
        assert abs(m.G["g"][0].item() - G["g"]) <= de.sum() + gam(B + 1) * np.abs(e).sum() * 2
    for k in m.G:
        m.G[k].zero_()


@pytest.mark.parametrize("name", ["MF", "PMF", "FM"])
@pytest.mark.parametrize("f", [1, 4, 10, 50, 128])
def test_mse_steps_match_fp64(name, f):
    nu, ni = 300, 500
    indptr, indices = _csr(nu, ni, f)
    m = _model(name, nu, ni, f, indptr, indices)
    rs = np.random.RandomState(f)
    for B in (1, 512, 4096):
        _check_mse_step(m, name, f, *_batch(rs, nu, ni, B, name))


def test_pmf_saturated_sigmoid():
    nu, ni, f = 50, 60, 8
    indptr, indices = _csr(nu, ni, 1)
    m = _model("PMF", nu, ni, f, indptr, indices)
    m.P["P"][:, :f] = 3.0; m.P["Q"][:10, :f] = 3.0; m.P["Q"][10:, :f] = -3.0  # logits +-72: sigmoid 1 or ~5e-32
    rs = np.random.RandomState(0)
    u, it, y = _batch(rs, nu, ni, 512, "PMF")
    _check_mse_step(m, "PMF", f, u, it, y)


def _lmf_step_check(m, f, u, it, y):
    T = _host(m, "LMF", f)
    u64 = u.astype(np.int64)
    a, lam = m.alpha, m.reg
    loss_ref, G, x = pm.lmf_forward_backward(T, u64, it, y.astype(np.float64), a, lam)
    S = np.abs(T["Gu"][u64] * T["Gi"][it]).sum(1) + np.abs(T["Bu"][u64]) + np.abs(T["Bi"][it])
    dx = gam(f + 2) * S
    ay = a * y
    c = pm.sigmoid(x) * (1 + ay) - ay
    dc = dx * (1 + ay) / 4 + 8 * U32 * (1 + ay)
    before = {k: m.P[k].clone() for k in ("Gu", "Bu")}
    m._loss.zero_()
    m.grads((d(u), d(it), d(y)))
    torch.cuda.synchronize()
    sq = (T["Gu"][u64] ** 2).sum(1) + (T["Gi"][it] ** 2).sum(1)
    Lterm = np.abs(ay * x) + (1 + ay) * pm.softplus(x)
    loss_bound = (np.abs(c) * dx + 8 * U32 * Lterm + lam / 2 * gam(2 * f + 2) * sq).sum() + gam(len(u)) * 0
    assert np.isfinite(m._loss.item()) and abs(m._loss.item() - loss_ref) <= loss_bound + 1e-12 * abs(loss_ref)
    mult = np.bincount(it).max()
    contrib = np.abs(c)[:, None] * np.abs(T["Gu"][u64]) + lam * np.abs(T["Gi"][it])
    bound = _scatter_abs(ni := T["Gi"].shape[0], it, np.abs(T["Gu"][u64]) * dc[:, None]) + (2 * U32 + gam(mult)) * _scatter_abs(ni, it, contrib)
    got = m.G["Gi"][:, :f].double().cpu().numpy()
    assert np.isfinite(got).all() and (np.abs(got - G["Gi"]) <= bound + 1e-30).all()
    bb = _scatter_abs(ni, it, dc) + gam(mult) * _scatter_abs(ni, it, c)
    assert (np.abs(m.G["Bi"].double().cpu().numpy() - G["Bi"]) <= bb + 1e-30).all()
    for k in before:                                                     # no user row is ever written
        assert torch.equal(m.P[k], before[k])


@pytest.mark.parametrize("f", [2, 4, 10, 50, 128])
def test_lmf_step_matches_fp64(f):
    nu, ni = 300, 500
    m = _model("LMF", nu, ni, f, None, None)
    rs = np.random.RandomState(f)
    for B in (1, 512, 4096):
        _lmf_step_check(m, f, *_batch(rs, nu, ni, B, "LMF"))
        m.G["Gi"].zero_(); m.G["Bi"].zero_()


def test_lmf_step_finite_beyond_softplus_overflow():
    nu, ni, f = 40, 50, 8
    m = _model("LMF", nu, ni, f, None, None)
    m.P["Gu"][:20, :f] = 4.0; m.P["Gu"][20:, :f] = -4.0; m.P["Gi"][:, :f] = 4.0   # x = +-128 (+ biases): |x| > 90
    rs = np.random.RandomState(1)
    u, it, y = _batch(rs, nu, ni, 512, "LMF")
    _lmf_step_check(m, f, u, it, y)


def test_lmf_training_leaves_users_bit_identical():
    nu, ni, f = 100, 200, 10
    m = _model("LMF", nu, ni, f, None, None)
    Gu, Bu = m.P["Gu"].clone(), m.P["Bu"].clone()
    Gi = m.P["Gi"].clone()
    rs = np.random.RandomState(2)
    for _ in range(5):
        m.train_step(tuple(d(a) for a in _batch(rs, nu, ni, 512, "LMF")))
    torch.cuda.synchronize()
    assert torch.equal(m.P["Gu"], Gu) and torch.equal(m.P["Bu"], Bu) and not torch.equal(m.P["Gi"], Gi)
    assert set(m.acc) == {"Gi", "Bi"} and set(m.G) == {"Gi", "Bi"}     # no user-side state exists


def test_adagrad_rows():
    n, ld, width, lr, eps = 400, 16, 10, 0.05, 1e-7
    rs = np.random.RandomState(5)
    var = d(rs.randn(n, ld).astype(np.float32)); acc = d((0.1 + rs.rand(n, ld)).astype(np.float32))
    bvar = d(rs.randn(n).astype(np.float32)); bacc = d((0.1 + rs.rand(n)).astype(np.float32))
    rows = np.r_[rs.randint(0, n, 300), [7, 7, 7, 7, 9, 9]].astype(np.int32)
    grad = torch.zeros_like(var); bgrad = torch.zeros_like(bvar)
    touched = np.unique(rows)
    grad[d(touched.astype(np.int64))] = d(rs.randn(len(touched), ld).astype(np.float32))
    bgrad[d(touched.astype(np.int64))] = d(rs.randn(len(touched)).astype(np.float32))
    grad[:, width:] = 0
    h = {k: t.double().cpu().numpy() for k, t in dict(var=var, acc=acc, grad=grad, bvar=bvar, bacc=bacc, bgrad=bgrad).items()}
    stamp = torch.zeros(n, dtype=torch.int64, device=DEV)
    for step in (1, 2):                                                  # the second step: same rows, zero gradients
        v0, a0, bv0, ba0 = var.clone(), acc.clone(), bvar.clone(), bacc.clone()
        ops.adagrad_rows_f32(var, acc, grad, d(rows), stamp, step, lr, width=width, bvar=bvar, bacc=bacc, bgrad=bgrad, eps=eps)
        torch.cuda.synchronize()
        assert not grad.any() and not bgrad.any()                        # every touched gradient cleared
        if step == 2:                                                    # zero gradients leave every value as it was
            assert torch.equal(var, v0) and torch.equal(acc, a0) and torch.equal(bvar, bv0) and torch.equal(bacc, ba0)
    untouched = np.setdiff1d(np.arange(n), touched)
    for k, t in (("var", var), ("acc", acc), ("bvar", bvar), ("bacc", bacc)):
        assert np.array_equal(t.double().cpu().numpy()[untouched], h[k][untouched]), k   # bit-identical
    for (vk, ak, gk, cols) in (("var", "acc", "grad", slice(0, width)), ("bvar", "bacc", "bgrad", slice(None))):
        v, a = h[vk].copy(), h[ak].copy()
        g = h[gk]
        pm.adagrad_dense(v, a, g, lr, eps)                               # once per row, though 7 and 9 repeat
        gv, ga = (var if vk == "var" else bvar).double().cpu().numpy(), (acc if vk == "var" else bacc).double().cpu().numpy()
        step_mag = np.abs(lr * g / (np.sqrt(a) + eps))
        assert (np.abs(ga - a)[touched][..., cols] <= 3 * U32 * a[touched][..., cols]).all(), ak
        assert (np.abs(gv - v)[touched][..., cols] <= 8 * U32 * step_mag[touched][..., cols]
                + U32 * np.abs(v[touched][..., cols])).all(), vk
    assert np.array_equal(var.double().cpu().numpy()[:, width:], h["var"][:, width:])   # past `width`: untouched


def test_mf_null_bias_path_equals_explicit_zero_biases():
    """The null-bias form gives exactly what zero bias tables give (adding 0.f is exact)."""
    nu, ni, f = 200, 300, 12
    indptr, indices = _csr(nu, ni, 3)
    m = _model("MF", nu, ni, f, indptr, indices)
    rs = np.random.RandomState(3)
    u, it, y = (d(a) for a in _batch(rs, nu, ni, 700, "MF"))
    P = m.P
    dP1, dQ1 = torch.zeros_like(P["P"]), torch.zeros_like(P["Q"])
    dP2, dQ2 = torch.zeros_like(P["P"]), torch.zeros_like(P["Q"])
    zu, zi = torch.zeros(nu, device=DEV), torch.zeros(ni, device=DEV)
    l1, l2 = (torch.zeros(1, dtype=torch.float64, device=DEV) for _ in range(2))
    ops.rating_mf_step_f32(P["P"], P["Q"], None, None, None, m.fp, u, it, y, dP1, dQ1, None, None, None, loss=l1)
    ops.rating_mf_step_f32(P["P"], P["Q"], zu, zi, None, m.fp, u, it, y, dP2, dQ2, torch.zeros_like(zu), torch.zeros_like(zi), None,
                           loss=l2)
    torch.cuda.synchronize()
    assert abs(l1.item() - l2.item()) <= 1e-12 * l2.item()
    assert torch.allclose(dQ1, dQ2, rtol=1e-6, atol=1e-9) and torch.allclose(dP1, dP2, rtol=1e-6, atol=1e-9)
    _check_mse_step(m, "MF", f, *_batch(rs, nu, ni, 512, "MF"))


def test_rating_labels_pass():
    nu, ni = 150, 400
    indptr, indices = _csr(nu, ni, 4)
    ratings = np.random.RandomState(5).randint(1, 6, indices.size).astype(np.float32)
    n = 100000
    u, i, y = ops.pointwise_sample_philox(nu, ni, d(indptr), d(indices), n, 42)
    y0 = y.clone()
    ops.rating_labels_(d(indptr), d(indices), d(ratings), u, i, y)
    u, i, y, y0 = (t.cpu().numpy() for t in (u, i, y, y0))
    assert np.array_equal(y, pm.rating_labels(indptr, indices, ratings.astype(np.float64), u, i, y0).astype(np.float32))
    pos = y0 != 0
    assert 0.45 < pos.mean() < 0.55 and (y[pos] >= 1).all() and (y[~pos] == 0).all()
    for s in np.flatnonzero(~pos)[:5000]:                                # negatives are not in the train row
        assert i[s] not in indices[indptr[u[s]]:indptr[u[s] + 1]]


@pytest.mark.parametrize("name", ["MF", "PMF", "FM"])
def test_train_step_is_one_keras_adam_step(name):
    nu, ni, f = 200, 300, 10
    indptr, indices = _csr(nu, ni, 1)
    m = _model(name, nu, ni, f, indptr, indices)
    rs = np.random.RandomState(2)
    u, it, y = _batch(rs, nu, ni, 500, name)
    T = _host(m, name, f)
    fn = {"MF": pm.mf_forward_backward, "PMF": pm.pmf_forward_backward, "FM": pm.fm_forward_backward}[name]
    _, G, _ = fn(T, u.astype(np.int64), it, y.astype(np.float64))
    opt = tfm.KerasAdam(1e-3); opt.begin_step()
    want = {k: np.array(v, np.float64) for k, v in T.items()}
    for k in want:
        opt.apply(k, want[k], np.asarray(G[k], np.float64))
    m.train_step((d(u), d(it), d(y)))
    after = _host(m, name, f)
    for k in want:
        assert np.abs(np.asarray(after[k]) - want[k]).max() < 2e-6, k
    assert not m.P["P"][:, f:].any() and not m.P["Q"][:, f:].any()
    assert set(m.P) == {"MF": {"P", "Q"}, "PMF": {"P", "Q"}, "FM": {"P", "Q", "bu", "bi", "g"}}[name]


@pytest.mark.parametrize("name", ["MF", "PMF", "FM", "LMF"])
@pytest.mark.parametrize("k", [10, 50])
def test_topk_against_fp64(name, k):
    nu, ni, f = 400, 900, 10
    indptr, indices = _csr(nu, ni, 9)
    m = _model(name, nu, ni, f, indptr, indices)
    mp, mi = d(indptr), d(indices)
    idx, val = m.topk(k, mp, mi)
    U, V = (m.P["Gu"], m.P["Gi"]) if name == "LMF" else (m.P["P"], m.P["Q"])
    bias = m.P["Bi"] if name == "LMF" else m.P.get("bi")
    if k <= 16:
        raw_idx, raw_val, _ = ops.score_topk_tc(U, V, bias, f, k, mp, mi, stats=False)
    else:
        raw_idx, raw_val = ops.score_topk(U, V, bias, f, k, mp, mi)
    filled, total = check_topk_fp64(U[:, :f].double().cpu().numpy(), V[:, :f].double().cpu().numpy(),
                                    None if bias is None else bias[:ni].double().cpu().numpy(), f, k, indptr, indices,
                                    np.arange(nu), idx.cpu().numpy(), raw_val.cpu().numpy(), U32)
    assert total > 0 and filled > 0 and np.array_equal(idx.cpu().numpy(), raw_idx.cpu().numpy())
    T = _host(m, name, f)
    full = pm.full_scores(name, T)
    ok = idx.cpu().numpy() >= 0
    want = np.take_along_axis(full, np.maximum(idx.cpu().numpy(), 0).astype(np.int64), 1)
    v = val.double().cpu().numpy()
    S = np.abs(U[:, :f].double().cpu().numpy()) @ np.abs(V[:, :f].double().cpu().numpy()).T
    tol = np.take_along_axis(S, np.maximum(idx.cpu().numpy(), 0).astype(np.int64), 1) * gam(f + 3) + 1e-6
    assert (np.abs(v - want)[ok] <= tol[ok]).all()                       # the kept values are the model's full-list scores


def _small_data():
    import pandas as pd
    from elliot_b200.dataset import DataSet
    rs = np.random.RandomState(8)
    rows = []
    for u in range(60):
        its = rs.choice(80, size=rs.randint(8, 30), replace=False)
        rows += [(u + 1, i + 1, float(rs.randint(1, 6))) for i in its]
    rows = np.array(rows)
    test = rs.rand(len(rows)) < 0.3
    te = np.r_[rows[test], [(3, 999, 5.0), (9, 998, 4.0)], [rows[~test][0][:2].tolist() + [5.0]]]   # test-only; one train item
    frame = lambda a: pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})
    cfg = SimpleNamespace(config_test=True, top_k=10, evaluation=SimpleNamespace(
        simple_metrics=["nDCG", "MAE", "MSE", "RMSE", "AUC"], relevance_threshold=0, paired_ttest=False, cutoffs=[5, 10]))
    return DataSet(cfg, (frame(rows[~test]), frame(te)))


@pytest.mark.parametrize("name", ["MF", "PMF", "FM", "LMF"])
def test_pair_and_rank_passes(name):
    from elliot_b200.dataset import train_csr_of
    from elliot_b200.evaluation import Evaluator
    data = _small_data()
    indptr, _, srt = train_csr_of(data, torch.device(DEV), set_order=False)
    m = _model(name, data.num_users, data.num_items, 12, indptr.cpu().numpy(), srt.cpu().numpy())
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), rank_pass=True, score_pass=True)
    rel_indptr, rel_items, _ = ev.pair_sets(torch.device(DEV))["test"]
    s = m.pair_scores(rel_indptr, rel_items, indptr, srt).cpu().numpy()
    idx, val = m.topk(data.num_items, indptr, srt)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    rp, ri = rel_indptr.cpu().numpy(), rel_items.cpu().numpy()
    train = [set(srt[indptr[u]:indptr[u + 1]].cpu().numpy().tolist()) for u in range(data.num_users)]
    full = pm.full_scores(name, _host(m, name, 12))
    n_inf = n_nan = 0
    for u in range(data.num_users):
        ok = idx[u] >= 0
        listed = dict(zip(idx[u][ok].tolist(), val[u][ok].tolist()))
        for e in range(rp[u], rp[u + 1]):
            it = int(ri[e])
            if it < 0:
                assert np.isnan(s[e]); n_nan += 1                        # outside the catalogue: NaN, also for PMF
            elif it in train[u]:
                assert np.isneginf(s[e]); n_inf += 1                     # a train item: -inf, also after PMF's sigmoid
            else:
                assert abs(s[e] - listed[it]) <= 4e-7 * max(1.0, abs(listed[it]))
                assert abs(s[e] - full[u, it]) <= 1e-5
    assert n_inf == 1 and n_nan == 2
    # rank pass: per relevant entry, the non-relevant non-train items ahead of it in the fp64 full list (ties excluded)
    n_pos, sum_c = (t.cpu().numpy() for t in m.rank(rel_indptr, rel_items, indptr, srt))
    for u in range(data.num_users):
        rel = set(ri[rp[u]:rp[u + 1]].tolist())
        cand = [j for j in range(data.num_items) if j not in train[u] and j not in rel]
        pos = [j for j in rel if j >= 0 and j not in train[u]]
        assert n_pos[u] == len(pos)
        lo = sum(sum(full[u, j] > full[u, p] + 1e-5 for j in cand) for p in pos)
        hi = sum(sum(full[u, j] > full[u, p] - 1e-5 for j in cand) for p in pos)
        assert lo <= sum_c[u] <= hi


C1_BLOCK = {"epochs": 4, "factors": 10, "lr": 0.01, "reg": 0.1, "seed": 7}


@pytest.fixture(scope="module")
def c1_tsv(tmp_path_factory):
    d_ = tmp_path_factory.mktemp("pointwise_c1")
    tsv = str(d_ / "dataset.tsv")
    synth_c1.write_tsv(tsv)
    return tsv


def _c1_yaml(tsv, out, key, meta, batch, device_eval=False):
    block = dict(C1_BLOCK, batch_size=batch, meta=meta, **({"b200_eval": "device"} if device_eval else {}))
    if key.endswith("LMF"):
        block["alpha"] = 0.5
    text = synth_c1.experiment_yaml(tsv, out, key, "", metrics=("nDCG", "MAE", "RMSE", "AUC"), meta=())
    cfg = yaml.safe_load(text)
    if key.startswith("external."):
        import os
        cfg["experiment"]["external_models_path"] = os.path.join(os.path.dirname(synth_c1.__file__), "plugin.py")
    cfg["experiment"]["models"] = {key: block}
    return yaml.safe_dump(cfg)


@pytest.mark.parametrize("batch", [512, -1])
@pytest.mark.parametrize("key", ["MF", "PMF", "FM", "LMF", "external.MF", "external.LMF"])
def test_c1_run_trains_saves_and_restores(c1_tsv, tmp_path, key, batch):
    from elliot_b200 import run_experiment
    from elliot_b200.recommender import logistic_mf, rating_mf
    if key.startswith("external.") and batch != 512:
        pytest.skip("the external form is checked at one batch size")
    losses = []
    owner = logistic_mf.LMF if key.endswith("LMF") else rating_mf._RatingMF
    orig = owner.train

    def recording_train(self):                                          # pass-through: keeps the epoch losses
        out = orig(self)
        losses.extend(self._losses)
        return out
    owner.train = recording_train
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"save_weights": True, "save_recs": False}, batch))
        res = run_experiment(str(p))[0]
    finally:
        owner.train = orig
    short = key.split(".")[-1]
    hist = res["history"]
    assert len(hist) == 4 and res["name"].startswith(short + "_")
    for h in hist:
        assert all(np.isfinite(h[10][m]) for m in ("nDCG", "MAE", "RMSE", "AUC"))
    epoch_sums = [l * (e + 1) for e, l in enumerate(losses)]             # evaluate() gets the epoch sum / (epoch + 1)
    assert epoch_sums[-1] < epoch_sums[0], epoch_sums
    best = res["test_results"][10]
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"restore": True, "save_recs": False}, batch))
    again = run_experiment(str(p))[0]["test_results"][10]
    for m in ("nDCG", "MAE", "RMSE", "AUC"):
        assert again[m] == best[m], m
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"restore": True, "save_recs": False}, batch, device_eval=True))
    dev = run_experiment(str(p))[0]["test_results"][10]
    for m in ("nDCG", "MAE", "RMSE", "AUC"):
        assert dev[m] == best[m] or abs(dev[m] - best[m]) <= 1e-12 * abs(best[m]), m


@pytest.mark.parametrize("key,params,err,match", [
    ("MF", {"factors": 0}, ValueError, "outside"), ("PMF", {"factors": 129}, ValueError, "outside"),
    ("FM", {"factors": 200}, ValueError, "outside"), ("LMF", {"factors": 129}, ValueError, "outside"),
    ("LMF", {"factors": 1}, ValueError, "factors=1"), ("FM", {"loader": "Feats"}, NotImplementedError, "side information")])
def test_refusals(c1_tsv, tmp_path, monkeypatch, key, params, err, match):
    from elliot_b200 import run_experiment
    from elliot_b200.dataset import DataSet
    if "loader" in params:                                               # a loader carrying item features
        orig = DataSet.__init__

        def with_features(self, *a, **k):
            orig(self, *a, **k)
            self.side_information.Feats = SimpleNamespace(nfeatures=3, feature_map={})
        monkeypatch.setattr(DataSet, "__init__", with_features)
    p = tmp_path / "cfg.yml"
    text = _c1_yaml(c1_tsv, str(tmp_path), key, {"save_recs": False}, 512)
    cfg = yaml.safe_load(text)
    cfg["experiment"]["models"][key].update(params, epochs=1)
    p.write_text(yaml.safe_dump(cfg))
    with pytest.raises(err, match=match):
        run_experiment(str(p))
