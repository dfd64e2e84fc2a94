"""GPU tests of CML (csrc/cml.cu, recommender/cml.py): the step against the fp64 restatements of oracle/cml.py (the literal
B x B broadcast up to B = 4096, the counting form at the C1 batch of every transaction), one Keras Adam step, the top-k
against the fp64 direct form, the AUC / GAUC rank pass against the host formula, and C1 runs through run_experiment."""
import numpy as np
import pytest
import torch
import yaml

from elliot_b200 import ops, synth_c1
from oracle import auc as auc_oracle
from oracle import cml as oracle
from oracle import tf_models as tfm
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 2.0 ** -24
H = 1 / 8                        # bias grid: E_b on multiples of H
M_GRID = 0.5 + H / 2             # a margin halfway between grid points


def _model(nu, ni, f, margin=0.5, lr=1e-3, seed=3):
    from elliot_b200.recommender.cml import CMLModel
    return CMLModel(f, lr, 0.01, 0.02, margin, nu, ni, seed, DEV)


def _set(m, Gu, Gi, Bi):
    f = Gu.shape[1]
    m.Gu.zero_(); m.Gu[:, :f] = torch.from_numpy(Gu).float().to(DEV)
    m.Gi.zero_(); m.Gi[:, :f] = torch.from_numpy(Gi).float().to(DEV)
    m.Bi.zero_(); m.Bi[:len(Bi)] = torch.from_numpy(Bi).float().to(DEV)


def _host(m):
    f, ni = m._factors, m._num_items
    return (m.Gu[:, :f].double().cpu().numpy(), m.Gi[:, :f].double().cpu().numpy(), m.Bi[:ni].double().cpu().numpy())


def _grid_tables(rs, nu, ni, f, scale):
    """Rows small enough that |D_a| < H/2 - 1e-4, biases on the grid H, items 0 and 1 at -90 (their pairs fall below
    -80): with the margin M_GRID every pair lies at least 1e-4 from -80 and from the margin."""
    Gu = rs.uniform(-scale, scale, (nu, f)).astype(np.float32)
    Gi = rs.uniform(-scale, scale, (ni, f)).astype(np.float32)
    Bi = (rs.randint(-8, 9, ni) * H).astype(np.float32)
    Bi[0] = Bi[1] = -90.0
    return Gu, Gi, Bi


def _triples(rs, B, nu, ni):
    u = rs.randint(0, nu, B).astype(np.int32); i = rs.randint(0, ni, B).astype(np.int32)
    j = rs.randint(0, ni, B).astype(np.int32)
    u[: B // 4] = 5; i[B // 8: B // 3] = 7; j[B // 2: B // 2 + B // 5] = 7         # repeated rows
    k = rs.choice(B, size=max(1, B // 16), replace=False)
    i[k[::2]] = 0; j[k[1::2]] = 1                                                    # pairs below -80 and far above m
    return u, i, j


def _dev(*a):
    return tuple(torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in a)


def _bounds(Gu, Gi, Bi, u, i, j, n_a, n_b, l_w, l_b):
    """Per-element bounds of the fp32 step against exact arithmetic on its inputs.  Each term of a gradient row is
    c (x - y) + l_w z with c = 2 n_a exact: three roundings, 3 unit (|c (x - y)| + |l_w z|); k terms of a row are summed
    by atomics in any order, gamma(k) times their absolute sum: (k + 3) unit in all.  The bias terms -n'_b + l_b b are
    one rounding each, (k + 2) unit.  D_a is two d-term fp32 sums of squared differences and one subtraction:
    (d + 4) unit (p_a + q_a); E_b one subtraction: unit |E_b|.  The hinge sum moves by at most n_a |dD_a| + n'_b |dE_b|
    per triple, the l2 terms by (3d + 3) unit of their value, and the fp64 sums by 1e-12 of the loss."""
    d = Gu.shape[1]
    gu, gp, gn, bp, bn = Gu[u], Gi[i], Gi[j], Bi[i], Bi[j]
    na = 2.0 * n_a[:, None]
    p, q = ((gu - gp) ** 2).sum(1), ((gu - gn) ** 2).sum(1)
    out = {}
    for name, tab, rows, terms in (("Gu", Gu, u, [np.abs(na * (gp - gn)) + np.abs(l_w * gu)]),
                                   ("Gi", Gi, np.r_[i, j], [np.abs(na * (gu - gp)) + np.abs(l_w * gp),
                                                            np.abs(na * (gu - gn)) + np.abs(l_w * gn)])):
        s = np.zeros_like(tab); np.add.at(s, rows, np.concatenate(terms))
        k = np.bincount(rows, minlength=len(tab))[:, None]
        out[name] = (k + 3) * U32 * s
    s = np.zeros_like(Bi); np.add.at(s, np.r_[i, j], np.r_[n_b + np.abs(l_b * bp), n_b + np.abs(l_b * bn / 10)])
    out["Bi"] = (np.bincount(np.r_[i, j], minlength=len(Bi)) + 2) * U32 * s
    dD = (d + 4) * U32 * (p + q)
    dE = U32 * np.abs(bp - bn)
    reg = l_w * ((gu ** 2).sum() + (gp ** 2).sum() + (gn ** 2).sum()) / 2 + l_b * ((bp ** 2).sum() / 2 + (bn ** 2).sum() / 20)
    out["loss"] = (n_a * dD).sum() + (n_b * dE).sum() + (3 * d + 3) * U32 * reg
    out["D"], out["E"] = dD, dE
    return out


def _check_step(m, u, i, j, want, extra_loss_tol=0.0):
    """The device step on (u, i, j) against `want` = (loss, dGu, dGi, dBi, n_a, n'_b) of the restatement on the same
    fp64-widened tables; returns the device terms."""
    Gu, Gi, Bi = _host(m)
    B = len(u)
    terms = torch.empty(2 * B, dtype=torch.float32, device=DEV)
    m.grads(_dev(u, i, j), terms=terms)
    torch.cuda.synchronize()
    bd = _bounds(Gu, Gi, Bi, u, i, j, want[4], want[5], m._l_w, m._l_b)
    loss = float(m._loss.item())
    assert abs(loss - want[0]) <= bd["loss"] + 1e-12 * abs(want[0]) + extra_loss_tol, (loss, want[0], bd["loss"])
    f = m._factors
    got = {"Gu": m.grad["Gu"], "Gi": m.grad["Gi"], "Bi": m.grad["Bi"][:m._num_items]}
    for name, w in zip(("Gu", "Gi", "Bi"), want[1:4]):
        g = got[name].double().cpu().numpy()
        if name != "Bi":
            assert not g[:, f:].any(), "padding columns got a gradient"
            g = g[:, :f]
        err = np.abs(g - w)
        assert (err <= bd[name] + 1e-30).all(), f"{name}: off by {(err / np.maximum(bd[name], 1e-30)).max():.3g} bounds"
    assert not m.grad["Bi"][m._num_items:].any()
    D, E = terms[:B].double().cpu().numpy(), terms[B:].double().cpu().numpy()
    D64, E64 = oracle.terms(Gu, Gi, Bi, u, i, j)
    assert (np.abs(D - D64) <= bd["D"]).all() and (np.abs(E - E64) <= bd["E"]).all()
    return D, E


@pytest.mark.parametrize("f,B", [(2, 4096), (5, 300), (16, 1), (16, 2), (64, 4096), (100, 4096), (256, 1000)])
def test_step_matches_broadcast_restatement(f, B):
    nu, ni = 300, 500
    rs = np.random.RandomState(f * 7 + B)
    m = _model(nu, ni, f, margin=M_GRID)
    Gu, Gi, Bi = _grid_tables(rs, nu, ni, f, scale=0.08 / f ** 0.25)
    _set(m, Gu, Gi, Bi)
    u, i, j = _triples(rs, B, nu, ni)
    if B <= 2:                                                          # one pair in range; at B = 2 one below -80
        i[:], j[:] = np.array([9, 0])[:B], 11
    Gu, Gi, Bi = _host(m)
    D64, E64 = oracle.terms(Gu, Gi, Bi, u, i, j)
    x = D64[:, None] + E64[None, :]
    assert np.abs(D64).max() < H / 2 - 1e-4
    assert np.abs(x - M_GRID).min() >= 1e-4 and np.abs(x + 80).min() >= 1e-4
    want = oracle.broadcast_step(Gu, Gi, Bi, u, i, j, m._l_w, m._l_b, float(np.float32(M_GRID)))
    if B >= 300:
        assert 0 < want[4].sum() < B * B and (x < -80).any()
    _check_step(m, u, i, j, want)


def test_step_ties_at_margin_and_clip():
    """Dyadic tables: every fp32 and fp64 sum is exact, so pairs sit exactly on m (active: Maximum's tie) and on -80
    (inactive: the clip's bound), and the step equals the restatement up to the atomics' order."""
    nu, ni, f, B = 30, 40, 4, 600
    rs = np.random.RandomState(1)
    m = _model(nu, ni, f, margin=0.5)
    Gu = (rs.randint(-2, 3, (nu, f)) / 8.0).astype(np.float32); Gi = (rs.randint(-2, 3, (ni, f)) / 8.0).astype(np.float32)
    Bi = (rs.randint(-32, 33, ni) / 64.0).astype(np.float32); Bi[0] = -80.0; Bi[1] = -90.0
    _set(m, Gu, Gi, Bi)
    u, i, j = _triples(rs, B, nu, ni)
    Gu, Gi, Bi = _host(m)
    D64, E64 = oracle.terms(Gu, Gi, Bi, u, i, j)
    x = D64[:, None] + E64[None, :]
    assert (x == 0.5).sum() > 0 and (x == -80.0).sum() > 0
    want = oracle.broadcast_step(Gu, Gi, Bi, u, i, j, m._l_w, m._l_b, 0.5)
    D, E = _check_step(m, u, i, j, want)
    assert np.array_equal(D, D64) and np.array_equal(E, E64)


def test_keras_adam_step_and_untouched_rows():
    """Two steps: the tables after each equal Keras Adam (fp64) fed the kernel's own gradient; rows outside the first
    batch do not move, and rows outside the second move only by the decayed moments of the first."""
    nu, ni, f = 200, 300, 20
    rs = np.random.RandomState(5)
    m = _model(nu, ni, f, lr=0.01)
    opt = tfm.KerasAdam(0.01)
    T = {k: v.double().cpu().numpy() for k, v in (("Gu", m.Gu), ("Gi", m.Gi), ("Bi", m.Bi))}
    for step, (lo, hi) in enumerate(((0, 100), (100, 200))):
        B = 700
        u = rs.randint(lo, hi, B).astype(np.int32)
        i = rs.randint(lo, hi, B).astype(np.int32); j = rs.randint(lo, hi, B).astype(np.int32)
        before = {k: t.clone() for k, t in (("Gu", m.Gu), ("Gi", m.Gi), ("Bi", m.Bi))}
        m.grads(_dev(u, i, j))
        G = {k: g.double().cpu().numpy() for k, g in m.grad.items()}
        m.adam()
        opt.begin_step()
        for k in ("Gu", "Gi", "Bi"):
            opt.apply(k, T[k], G[k])
            got = getattr(m, k).double().cpu().numpy()
            # fp32 Adam on the same gradient: a few roundings of the step (<= lr) and one of the variable
            assert np.abs(got - T[k]).max() <= 8 * U32 * (np.abs(T[k]).max() + 0.01), k
            T[k] = got                                                   # continue from the device's own state
        if step == 0:
            assert torch.equal(m.Gu[hi:], before["Gu"][hi:]) and torch.equal(m.Gi[hi:], before["Gi"][hi:])
            assert torch.equal(m.Bi[hi:], before["Bi"][hi:])
        else:
            moved = (m.Gu[:100] != before["Gu"][:100]).any(1)
            assert moved.float().mean() > 0.9                            # the decayed moments still move them


def test_step_at_c1_transactions_matches_sorted_restatement():
    """One batch of every C1 train transaction (the reference's default batch size), where the B x B matrix would
    take ~2.6 TB: the counting restatement on fp64 terms for grid tables, and on the kernel's own fp32 terms for the
    model's initial tables (the counts are then a function of those terms alone)."""
    nu, ni, f = synth_c1.N_USERS, synth_c1.N_ITEMS, 100
    B = 810_000
    rs = np.random.RandomState(11)
    m = _model(nu, ni, f, margin=M_GRID)
    Gu, Gi, Bi = _grid_tables(rs, nu, ni, f, scale=0.02)
    _set(m, Gu, Gi, Bi)
    u, i, j = _triples(rs, B, nu, ni)
    Gu, Gi, Bi = _host(m)
    D64, E64 = oracle.terms(Gu, Gi, Bi, u, i, j)
    assert np.abs(D64).max() < H / 2 - 1e-4
    want = oracle.sorted_step(Gu, Gi, Bi, u, i, j, m._l_w, m._l_b, float(np.float32(M_GRID)))
    assert 0 < want[4].sum() < B * B
    _check_step(m, u, i, j, want)
    del m
    # the model's own initial tables, margin 0.5: classify on the kernel's terms
    m2 = _model(nu, ni, f, margin=0.5)
    Gu, Gi, Bi = _host(m2)
    terms = torch.empty(2 * B, dtype=torch.float32, device=DEV)
    m2.grads(_dev(u, i, j), terms=terms)
    D, E = terms[:B].double().cpu().numpy(), terms[B:].double().cpu().numpy()
    want = oracle.sorted_step(Gu, Gi, Bi, u, i, j, m2._l_w, m2._l_b, 0.5, D=D, E=E)
    for t in m2.grad.values():
        t.zero_()
    # the fp64 loss of the restatement uses the kernel's D and E, so only the l2 terms and the sums' order differ
    _check_step(m2, u, i, j, want)


def _csr(rs, nu, ni):
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, 40), replace=False)) for _ in range(nu)]
    rows[1] = np.sort(rs.choice(ni, size=ni - 4, replace=False))          # runs out of candidates at k = 10
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


@pytest.mark.parametrize("k", [10, 50])
def test_topk_against_fp64_direct_form(k):
    nu, ni, f = 500, 1200, 24
    rs = np.random.RandomState(k)
    m = _model(nu, ni, f)
    _set(m, rs.normal(0, 0.3, (nu, f)).astype(np.float32), rs.normal(0, 0.3, (ni, f)).astype(np.float32),
         rs.normal(0, 0.5, ni).astype(np.float32))
    indptr, indices = _csr(rs, nu, ni)
    mp, mi = _dev(indptr, indices)
    idx, val = m.topk(k, mp, mi)
    U2, c, uo = m.score_operands()
    if k <= 16:
        raw_idx, raw_val, _ = ops.score_topk_tc(U2, m.Gi, c, f, k, mp, mi, stats=False)
    else:
        raw_idx, raw_val = ops.score_topk(U2, m.Gi, c, f, k, mp, mi)
    assert torch.equal(idx, raw_idx) and torch.equal(val, raw_val + uo[:, None])
    Gu, Gi, Bi = _host(m)
    assert torch.equal(U2[:, :f], 2 * m.Gu[:, :f]) and not U2[:, f:].any()
    # the scorer on its operands, under topk_bound's rules
    idx, val = idx.cpu().numpy(), val.double().cpu().numpy()
    filled, total = check_topk_fp64(U2.double().cpu().numpy(), Gi, c.double().cpu().numpy(), f, k, indptr, indices,
                                    np.arange(nu), idx, raw_val.cpu().numpy(), U32)
    assert total > 0 and filled > total // 2
    # the list values against the direct form Bi - |Gu - Gi|^2, and the returned set against its top k
    S = oracle.predict(Gu, Gi, Bi, 0, nu)
    for u in range(nu):
        S[u, indices[indptr[u]:indptr[u + 1]]] = -np.inf
    E = oracle.expansion_bound(Gu, Gi, Bi, np.arange(nu), U32)[:, None]
    got = idx >= 0
    assert not got.all() and np.isneginf(val[~got]).all()
    s = np.take_along_axis(S, np.where(got, idx, 0), 1)
    assert (np.where(got, np.abs(val - s), 0) <= E).all()
    top = -np.sort(-S, 1)[:, :k]
    srt = -np.sort(-np.where(got, s, -np.inf), 1)
    with np.errstate(invalid="ignore"):
        assert (np.where(got, np.abs(srt - top), 0) <= 2 * E).all()


def test_rank_pass_gives_host_auc_gauc():
    """Dyadic tables with a distinct low-order bias per item: every score is exact in fp32 and no two items tie, so the
    rank pass's counts must equal the fp64 full lists' exactly."""
    from elliot_b200.evaluation import finish_auc
    nu, ni, f = 300, 900, 8
    rs = np.random.RandomState(2)
    m = _model(nu, ni, f)
    Bi = rs.randint(-16, 17, ni) / 64.0 + np.arange(ni) * 2.0 ** -20
    _set(m, (rs.randint(-2, 3, (nu, f)) / 8.0).astype(np.float32), (rs.randint(-2, 3, (ni, f)) / 8.0).astype(np.float32),
         Bi.astype(np.float32))
    indptr, indices = _csr(rs, nu, ni)
    free = [np.setdiff1d(np.arange(ni), indices[indptr[u]:indptr[u + 1]]) for u in range(nu)]
    rel = [np.sort(rs.choice(c, size=min(rs.randint(0, 12), len(c)), replace=False)) for c in free]
    rp = np.r_[0, np.cumsum([len(r) for r in rel])].astype(np.int64)
    ri = np.concatenate(rel).astype(np.int32)
    n_pos, sum_c = (t.cpu().numpy() for t in m.rank(*_dev(rp, ri, indptr, indices)))
    Gu, Gi, Bi = _host(m)
    S = oracle.predict(Gu, Gi, Bi, 0, nu)
    lists, rels, train = {}, {}, {}
    for u in range(nu):
        tr = indices[indptr[u]:indptr[u + 1]]
        s = S[u].copy(); s[tr] = -np.inf
        assert len(np.unique(s[np.isfinite(s)])) == ni - len(tr)
        order = np.argsort(-s, kind="stable")
        lists[u] = order[: ni - len(tr)].tolist(); rels[u] = rel[u].tolist(); train[u] = len(tr)
        c = auc_oracle.rank_counts(lists[u], rels[u])
        assert (n_pos[u], sum_c[u]) == c[:2], u
    want = auc_oracle.auc_gauc(lists, rels, ni, train)
    got = finish_auc(n_pos, sum_c, np.diff(rp), np.diff(indptr), ni, ("AUC", "GAUC"))
    assert got["AUC"] == pytest.approx(want[0], rel=1e-14) and got["GAUC"] == pytest.approx(want[1], rel=1e-14)


def test_factors_below_two_refused():
    with pytest.raises(ValueError, match="factors >= 2"):
        _model(10, 10, 1)


# ---------------------------------------------------------------- C1 runs through run_experiment
@pytest.fixture(scope="module")
def c1_tsv(tmp_path_factory):
    tsv = str(tmp_path_factory.mktemp("cml_c1") / "dataset.tsv")
    synth_c1.write_tsv(tsv)
    return tsv


def _c1_yaml(tsv, out, block, meta, metrics=("nDCG", "AUC")):
    cfg = yaml.safe_load(synth_c1.experiment_yaml(tsv, out, "CML", "", metrics=metrics, meta=()))
    cfg["experiment"]["models"]["CML"] = dict(block, meta=meta)
    return yaml.safe_dump(cfg)


@pytest.mark.parametrize("batch", [512, -1])
def test_c1_run_trains_replays_sampler_saves_and_restores(c1_tsv, tmp_path, batch):
    from elliot_b200 import run_experiment
    from elliot_b200.recommender import cml
    block = {"epochs": 3, "batch_size": batch, "factors": 32, "lr": 0.001, "seed": 7}
    seen, models, lists = [], [], []
    orig_step, orig_train, orig_topk = cml.CMLModel.train_step, cml.CML.train, cml.CMLModel.topk

    def recording_step(self, batch_):                                  # pass-throughs: keep the triples, the model, the lists
        seen.append(tuple(t.cpu().numpy() for t in batch_))
        return orig_step(self, batch_)

    def recording_train(self):
        models.append(self)
        return orig_train(self)

    def recording_topk(self, *a, **kw):
        out = orig_topk(self, *a, **kw)
        lists.append(tuple(t.cpu().numpy() for t in out))
        return out
    cml.CMLModel.train_step, cml.CML.train, cml.CMLModel.topk = recording_step, recording_train, recording_topk
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), block, {"save_weights": True, "save_recs": False}))
        res = run_experiment(str(p))[0]
        trained = models[-1]
        n_trained_lists = len(lists)
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), block, {"restore": True, "save_recs": False}))
        again = run_experiment(str(p))[0]["test_results"][10]
    finally:
        cml.CMLModel.train_step, cml.CML.train, cml.CMLModel.topk = orig_step, orig_train, orig_topk
    assert res["name"].startswith("CML_") and len(res["history"]) == 3
    T = trained._data.transactions
    B = T if batch < 1 else batch
    assert len(seen) == 3 * ((T + B - 1) // B)
    # the triples consumed are MtSampler's stream from seed 42, epoch after epoch
    ref = ops.MtSampler(trained._num_users, trained._num_items, trained._indptr, trained._set_idx, trained._sorted_idx,
                        seed=42)
    per_epoch = len(seen) // 3
    for e in range(3):
        want = [t.cpu().numpy() for t in ref.step(T)]
        got = [np.concatenate([s[c] for s in seen[e * per_epoch:(e + 1) * per_epoch]]) for c in range(3)]
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    epoch_sums = [l * (e + 1) for e, l in enumerate(trained._losses)]   # evaluate() gets the epoch sum / (epoch + 1)
    assert all(np.isfinite(epoch_sums)) and epoch_sums[-1] < epoch_sums[0]
    best = res["test_results"][10]
    for name in ("nDCG", "AUC"):
        assert np.isfinite(best[name]) and again[name] == best[name], name
    # the restored model lists exactly what the trained one listed after the epoch whose weights were saved
    assert any(np.array_equal(lists[-1][0], a) and np.array_equal(lists[-1][1], b) for a, b in lists[:n_trained_lists])


def test_c1_rating_metrics_refused_before_training(c1_tsv, tmp_path):
    from elliot_b200 import run_experiment
    p = tmp_path / "cfg.yml"
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), {"epochs": 1, "factors": 8}, {"save_recs": False},
                         metrics=("nDCG", "MAE")))
    with pytest.raises(Exception, match="CML cannot evaluate MAE"):
        run_experiment(str(p))
