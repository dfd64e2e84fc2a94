"""GPU tests of DMF (csrc/dmf.cu, the pointwise ratio sampler in csrc/mt_sampler.cu, recommender/dmf.py): the device
sampler against the reference's goldens bit for bit, the towers, head and loss against the fp64 restatements of
oracle/dmf.py at bounds derived from the unit roundoff and the widths, one Keras Adam step, the block-normalised top-k
and the AUC / GAUC rank pass, and C1 runs through run_experiment."""
import os
import zlib

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import yaml

from elliot_b200 import ops, synth_c1
from oracle import dmf as oracle
from oracle import tf_models as tfm
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 2.0 ** -24
UBF = 2.0 ** -8                      # bf16 operand rounding (2^-9) plus the fp32 accumulation, per layer term
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _dev(a, dt=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)


def _sampler(indptr, rows, ratings, n_users, n_items, neg):
    srt = rows.copy()
    for u in range(n_users):
        srt[indptr[u]:indptr[u + 1]].sort()
    return ops.MtPointwiseRatioSampler(n_users, n_items, _dev(indptr), _dev(rows), _dev(ratings), _dev(srt), neg, seed=42)


# ---------------------------------------------------------------- sampler
@pytest.mark.parametrize("window", [None, 1, 37, 1000])
def test_sampler_matches_reference_goldens(window):
    g = np.load(os.path.join(GOLD, "dmf_sampler_cases.npz"))
    for name in g["names"]:
        n_users, n_items, neg, events, batch = (int(x) for x in g[f"{name}_meta"])
        s = _sampler(g[f"{name}_indptr"], g[f"{name}_rows"], g[f"{name}_ratings"], n_users, n_items, neg)
        for e in range(2):
            s.epoch()
            if window is None:                              # one call per reference batch, the list carried between them
                parts = [s.step(min(batch, events - a)) for a in range(0, events, batch)]
                u, i, r = (torch.cat([p[k] for p in parts]) for k in range(3))
            else:
                u, i, r = s.step(events, window=window)
            for got, key in ((u, "u"), (i, "i"), (r, "r")):
                assert np.array_equal(got.cpu().numpy(), g[f"{name}_e{e}_{key}"]), (name, e, key, window)


def _c1_rows():
    u, i, r = synth_c1.rows()
    d = {}
    for a, b, c in zip(u.tolist(), i.tolist(), r.tolist()):
        d.setdefault(a - 1, {})[b - 1] = float(c)
    rows = [list(set(d[k])) for k in range(len(d))]
    n_items = len({k for v in d.values() for k in v})
    indptr = np.r_[0, np.cumsum([len(x) for x in rows])].astype(np.int64)
    flat = np.concatenate(rows).astype(np.int32)
    rat = np.array([d[k][x] for k in range(len(d)) for x in rows[k]], np.float32)
    return (u, i, r), indptr, flat, rat, len(d), n_items


def test_sampler_c1_checksums_and_windows():
    g = np.load(os.path.join(GOLD, "dmf_sampler_c1.npz"))
    raw, indptr, flat, rat, n_users, n_items = _c1_rows()
    assert synth_c1.checksum(*raw) == int(g["checksum"])
    s = _sampler(indptr, flat, rat, n_users, n_items, int(g["neg_ratio"]))
    events = int(g["events"])
    for e in range(2):
        s.epoch()
        u, i, r = (t.cpu().numpy() for t in s.step(events))
        crc = [zlib.crc32(np.ascontiguousarray(u, np.int32).tobytes()), zlib.crc32(np.ascontiguousarray(i, np.int32).tobytes()),
               zlib.crc32(np.ascontiguousarray(r, np.float32).tobytes())]
        for k, s0 in enumerate(g["starts"]):
            w = g[f"e{e}_w{k}"]
            n = w.shape[1]
            assert np.array_equal(u[s0:s0 + n], w[0]) and np.array_equal(i[s0:s0 + n], w[1]) and np.array_equal(r[s0:s0 + n], w[2])
        assert crc == g[f"e{e}_crc"].tolist(), e


def test_sampler_refuses_user_owning_every_item():
    indptr = np.array([0, 2, 5], np.int64)
    rows = np.array([0, 1, 0, 1, 2], np.int32)
    s = _sampler(indptr, rows, np.ones(5, np.float32), 2, 3, 1)
    with pytest.raises(Exception, match="owns every item"):
        s.step(200)


# ---------------------------------------------------------------- towers, head, Adam
def _csr_data(rs, nu, ni, density=0.2):
    R = np.where(rs.rand(nu, ni) < density, rs.randint(1, 6, (nu, ni)), 0).astype(np.float32)
    R[np.arange(nu), rs.randint(0, ni, nu)] = 4.0
    Rs = sp.csr_matrix(R); Rs.sort_indices()
    Cs = sp.csr_matrix(R.T); Cs.sort_indices()
    up = lambda M: (_dev(M.indptr.astype(np.int64)), _dev(M.indices.astype(np.int32)), _dev(M.data.astype(np.float32)))
    return R.astype(np.float64), up(Rs), up(Cs)


def _model(nu, ni, umlp, imlp, sim, user_csr, item_csr, lr=1e-3, block=512, seed=3):
    from elliot_b200.recommender.dmf import DMFModel
    return DMFModel(nu, ni, umlp, imlp, sim, 5.0, lr, seed, DEV, user_csr, item_csr, block)


def _host_tower(t):
    n = len(t.widths)
    return [w.double().cpu().numpy() for w in t.W], [b.double().cpu().numpy()[:w] for b, w in zip(t.b, t.widths)], n


def _abs_chain(X, W, b):
    """Forward on absolute values: A_l >= |h_l| and the scale every rounding of layer l is taken against."""
    A, out = np.abs(X), []
    for l, w in enumerate(W):
        A = A @ np.abs(w if l == 0 else w.T) + np.abs(b[l])
        out.append(A)
    return out


def _fwd_bound(X, W, b, unit_dense):
    """fp32 sparse first layer (K0 = nnz of the row <= n_in terms, gamma(K0 + 1)), then each dense layer l with K_l terms
    at `unit_dense`; errors of earlier layers pass through |W| (first order): sum of (K_l + 2) units against the
    absolute-value chain."""
    A = _abs_chain(X, W, b)
    k0 = (X != 0).sum(1, keepdims=True) + 2
    tot = k0 * U32
    for l in range(1, len(W)):
        tot = tot + (W[l].shape[1] + 2) * unit_dense
    return tot * A[-1], A


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("sim", ["cosine", "dot"])
@pytest.mark.parametrize("B,umlp,imlp", [(1, [8], [8]), (64, [64, 32], [32, 32]), (300, [64, 32], [64, 32]),
                                         (4096, [128, 64, 16], [32, 16])])
def test_towers_head_and_gradients_match_fp64(exact, sim, B, umlp, imlp):
    nu, ni = 120, 200
    rs = np.random.RandomState(B + len(umlp))
    R, ucsr, icsr = _csr_data(rs, nu, ni)
    with ops.exact_gemm(exact):
        m = _model(nu, ni, umlp, imlp, sim, ucsr, icsr)
        if sim == "dot":                                   # outputs inside (0, 1) for a useful share of the batch
            for t in (m.user, m.item):
                t.W[0].mul_(20.0)
                t.b[-1][: t.widths[-1]] = 0.12
            m.user.refresh(); m.item.refresh()
        users = rs.randint(0, nu, B).astype(np.int32); items = rs.randint(0, ni, B).astype(np.int32)
        users[: B // 3] = 7; items[B // 4: B // 2] = 11              # repeated users and items
        ratings = np.where(rs.rand(B) < 0.4, R[users, items], 0.0).astype(np.float32)
        Uo = m.user.forward(_dev(users)); Vo = m.item.forward(_dev(items))
        Wu, bu, _ = _host_tower(m.user); Wi, bi, _ = _host_tower(m.item)
        unit = U32 if exact else UBF
        for out, X, W, b in ((Uo, R[users], Wu, bu), (Vo, R.T[items], Wi, bi)):
            want = oracle.tower(X, W, b)[0]
            bd, _ = _fwd_bound(X, W, b, unit)
            assert (np.abs(out.double().cpu().numpy() - want) <= bd + 1e-30).all()
        # head on the device's own tower outputs
        F = umlp[-1]
        U64, V64 = Uo.double().cpu().numpy(), Vo.double().cpu().numpy()
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        dU, dV = torch.empty_like(Uo), torch.empty_like(Vo)
        prob = torch.empty(B, device=DEV)
        ops.dmf_head_f32(Uo, Vo, F, _dev(ratings), 5.0, sim == "cosine", loss, dU, dV, prob=prob)
        wl, wdU, wdV, wo = oracle.head(U64, V64, ratings, 5.0, sim == "cosine")
        if sim == "cosine":
            uh, vh = oracle.l2_normalize_cols(U64)[0], oracle.l2_normalize_cols(V64)[0]
        else:
            uh, vh = U64, V64
        dO = (F + 4) * U32 * np.abs(uh * vh).sum(1)                      # F fp32 products and sums, the two scalings
        assert (np.abs(prob.double().cpu().numpy() - wo) <= dO).all()
        lo, hi = oracle.BCE_EPS, oracle.BCE_HI
        inside = (wo >= lo) & (wo <= hi)
        assert B < 64 or (inside.any() and (sim == "dot" or (~inside).any()))
        y = ratings.astype(np.float64) / 5.0
        p = np.clip(wo, lo, hi)
        g_all = -(y / (p + lo) - (1 - y) / (1 - p + lo)) / B
        g = np.where(inside, g_all, 0.0)
        # an output within dO of a clip bound may fall on either side of it on the device: its g is then 0 or g_all
        near = (np.abs(wo - lo) <= dO) | (np.abs(wo - hi) <= dO)
        dg = (np.where(inside, (y / (p + lo) ** 2 + (1 - y) / (1 - p + lo) ** 2) / B, 0.0) * dO + 4 * U32 * np.abs(g)
              + np.where(near, np.abs(g_all), 0.0))
        assert abs(loss.item() - wl) <= (np.abs(g) * dO).sum() + 1e-12 * abs(wl)
        for got, want, mine, other in ((dU, wdU, uh, vh), (dV, wdV, vh, uh)):
            if sim == "cosine":
                n = oracle.l2_normalize_cols(U64 if mine is uh else V64)[1]
                c = np.abs((g[:, None] * uh * vh).sum(0))
                dc = (dg[:, None] * np.abs(uh * vh)).sum(0) + 4 * U32 * (np.abs(g)[:, None] * np.abs(uh * vh)).sum(0)
                bd = n * (dg[:, None] * np.abs(other) + np.abs(mine) * dc + 8 * U32 * (np.abs(g)[:, None] * np.abs(other) + np.abs(mine) * c))
            else:
                bd = dg[:, None] * np.abs(other) + 2 * U32 * np.abs(g)[:, None] * np.abs(other)
            assert (np.abs(got.double().cpu().numpy() - want) <= bd + 1e-30).all()
        # tower backward from the device's own dU / dV
        m.user.backward(dU, m._grads_of(m.user)); m.item.backward(dV, m._grads_of(m.item))
        for t, X, W, b, d in ((m.user, R[users], Wu, bu, dU), (m.item, R.T[items], Wi, bi, dV)):
            _, pres, acts = oracle.tower(X, W, b)
            wW, wb = oracle.tower_backward(X, W, pres, acts, d.double().cpu().numpy())
            _, A = _fwd_bound(X, W, b, unit)
            G = m._grads_of(t)
            D = np.abs(d.double().cpu().numpy())
            depth = sum(W[l].shape[0] for l in range(1, len(W)))
            for l in range(len(W) - 1, -1, -1):
                inp = np.abs(X) if l == 0 else A[l - 1]
                absW = inp.T @ D if l == 0 else D.T @ inp
                k = (B + depth + 10) * (U32 if l == 0 and len(W) == 1 else unit)
                gw = G["W"][l].double().cpu().numpy()
                assert (np.abs(gw - wW[l]) <= k * absW + 1e-30).all(), (l, t is m.user)
                gb = G["b"][l][: t.widths[l]].double().cpu().numpy()
                assert (np.abs(gb - wb[l]) <= k * D.sum(0) + 1e-30).all(), (l, "bias")
                if l > 0:
                    D = D @ np.abs(W[l])


def test_adam_step_matches_keras():
    nu, ni = 60, 80
    rs = np.random.RandomState(4)
    R, ucsr, icsr = _csr_data(rs, nu, ni)
    m = _model(nu, ni, [32, 16], [32, 16], "cosine", ucsr, icsr, lr=0.01)
    opt = tfm.KerasAdam(0.01)
    T = [p.double().cpu().numpy() for p in m.P]
    for step in range(2):
        B = 256
        batch = (_dev(rs.randint(0, nu, B).astype(np.int32)), _dev(rs.randint(0, ni, B).astype(np.int32)),
                 _dev(rs.randint(0, 6, B).astype(np.float32)))
        m.grads(batch)
        G = [gr.double().cpu().numpy() for gr in m.G]
        m.adam()
        opt.begin_step()
        for k, (p, gr) in enumerate(zip(m.P, G)):
            opt.apply(k, T[k], gr)
            got = p.double().cpu().numpy()
            assert np.abs(got - T[k]).max() <= 8 * U32 * (np.abs(T[k]).max() + 0.01), (step, k)
            T[k] = got
        assert all(not gr.any() for gr in m.G)


# ---------------------------------------------------------------- scoring
def _mask(rs, nu, ni):
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, 30), replace=False)) for _ in range(nu)]
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


@pytest.mark.parametrize("k", [10, 50])
@pytest.mark.parametrize("sim,block", [("cosine", 64), ("cosine", 1000), ("dot", 64)])
def test_topk_matches_fp64_block_scores(k, sim, block):
    nu, ni = 300, 500                                                # 300 = 4 x 64 + a short block of 44
    rs = np.random.RandomState(k + block)
    R, ucsr, icsr = _csr_data(rs, nu, ni)
    m = _model(nu, ni, [64, 32], [64, 32], sim, ucsr, icsr, block=block)
    for t in (m.user, m.item):
        t.W[0].mul_(30.0)
    m.user.refresh(); m.item.refresh()
    indptr, indices = _mask(rs, nu, ni)
    idx, val = m.topk(k, _dev(indptr), _dev(indices))
    Uo, Vo = (t.double().cpu().numpy() for t in m.tower_outputs())
    Uh, Vh = oracle.score_operands(Uo, Vo, block, sim == "cosine")
    dUh, dVh, dVl = ops.dmf_score_operands_f32(*m.tower_outputs(), 32, block, sim == "cosine")
    bl = min(block, nu)
    # the device operands against fp64: a few roundings of each factor
    assert np.allclose(dUh[:, :32].double().cpu().numpy(), Uh, rtol=4 * U32, atol=1e-30)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    filled = total = 0
    for o in range(0, nu, bl):
        e = min(o + bl, nu)
        V = (dVl if (e - o) != bl and dVl is not None else dVh).double().cpu().numpy()
        assert np.allclose(V[:, :32], Vh[e - o], rtol=4 * U32, atol=1e-30)
        users = np.arange(o, e)
        f, t = check_topk_fp64(dUh.double().cpu().numpy(), V, None, 32, k, indptr, indices, users, idx[o:e], val[o:e], U32)
        filled += f; total += t
    assert total > 0 and filled > total // 2


def test_rank_pass_gives_fp64_auc_counts():
    """Each user's AUC counts from the rank pass: every relevant item counted, and the non-relevant items ahead of them
    between those surely ahead and those possibly ahead in the fp64 scores of the device operands (within the fp32
    dot products' rounding)."""
    nu, ni = 200, 300
    rs = np.random.RandomState(9)
    R, ucsr, icsr = _csr_data(rs, nu, ni)
    m = _model(nu, ni, [32, 16], [32, 16], "cosine", ucsr, icsr, block=64)
    for t in (m.user, m.item):
        t.W[0].mul_(30.0)
    m.user.refresh(); m.item.refresh()
    indptr, indices = _mask(rs, nu, ni)
    free = [np.setdiff1d(np.arange(ni), indices[indptr[u]:indptr[u + 1]]) for u in range(nu)]
    rel = [np.sort(rs.choice(c, size=min(rs.randint(0, 12), len(c)), replace=False)) for c in free]
    rp = np.r_[0, np.cumsum([len(r) for r in rel])].astype(np.int64)
    ri = np.concatenate(rel).astype(np.int32)
    n_pos, sum_c = (t.cpu().numpy() for t in m.rank(_dev(rp), _dev(ri), _dev(indptr), _dev(indices)))
    Uh, Vh, Vl = (None if t is None else t.double().cpu().numpy()
                  for t in ops.dmf_score_operands_f32(*m.tower_outputs(), 16, 64, True))
    for u in range(nu):
        V = Vl if u >= 192 else Vh
        s = V[:, :16] @ Uh[u, :16]
        bound = 2 * 20 * U32 * (np.abs(V[:, :16]) @ np.abs(Uh[u, :16]))      # 16-term fp32 dots on both sides, with margin
        s[indices[indptr[u]:indptr[u + 1]]] = -np.inf
        other = np.isfinite(s)
        other[rel[u]] = False
        lo = sum(int((s[other] > s[r] + bound[r] + bound[other]).sum()) for r in rel[u])
        hi = sum(int((s[other] >= s[r] - bound[r] - bound[other]).sum()) for r in rel[u])
        assert n_pos[u] == len(rel[u]) and lo <= sum_c[u] <= hi, u
    assert n_pos.sum() > 0 and sum_c.sum() > 0


def test_invalid_configurations_refused():
    nu, ni = 20, 30
    R, ucsr, icsr = _csr_data(np.random.RandomState(1), nu, ni)
    with pytest.raises(ValueError, match="multiple of 8"):
        _model(nu, ni, [64, 30], [64, 30], "cosine", ucsr, icsr)
    with pytest.raises(ValueError, match="same width"):
        _model(nu, ni, [64, 32], [64, 16], "cosine", ucsr, icsr)
    with pytest.raises(NotImplementedError):
        _model(nu, ni, [64, 32], [64, 32], "euclid", ucsr, icsr)


# ---------------------------------------------------------------- C1 runs through run_experiment
@pytest.fixture(scope="module")
def c1_tsv(tmp_path_factory):
    tsv = str(tmp_path_factory.mktemp("dmf_c1") / "dataset.tsv")
    synth_c1.write_tsv(tsv)
    return tsv


def _c1_yaml(tsv, out, block, meta, metrics=("nDCG", "AUC")):
    cfg = yaml.safe_load(synth_c1.experiment_yaml(tsv, out, "DMF", "", metrics=metrics, meta=()))
    cfg["experiment"]["models"]["DMF"] = dict(block, meta=meta)
    return yaml.safe_dump(cfg)


@pytest.mark.parametrize("batch,sim,epochs", [(512, "cosine", 2), (-1, "cosine", 3), (4096, "dot", 2)])
def test_c1_run_trains_replays_sampler_saves_and_restores(c1_tsv, tmp_path, batch, sim, epochs):
    from elliot_b200 import run_experiment
    from elliot_b200.recommender import dmf
    # at the full batch the column normalisation over ~6 M rows keeps every output near F / B, and a step of Adam moves
    # each weight by about lr: the reference's default lr keeps the step small enough to lower the loss
    block = {"epochs": epochs, "batch_size": batch, "lr": 0.001 if batch > 0 else 0.0001, "similarity": sim, "seed": 7}
    seen, running, models, lists = [], [], [], []
    orig_step, orig_train, orig_topk = dmf.DMFModel.train_step, dmf.DMF.train, dmf.DMFModel.topk

    def recording_step(self, batch_):
        seen.append(tuple(t.cpu().numpy() for t in batch_))
        out = orig_step(self, batch_)
        running.append(float(out.item()))                          # the epoch's running sum of batch losses
        return out

    def recording_train(self):
        models.append(self)
        return orig_train(self)

    def recording_topk(self, *a, **kw):
        out = orig_topk(self, *a, **kw)
        lists.append(tuple(t.cpu().numpy() for t in out))
        return out
    dmf.DMFModel.train_step, dmf.DMF.train, dmf.DMFModel.topk = recording_step, recording_train, recording_topk
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), block, {"save_weights": True, "save_recs": False}))
        res = run_experiment(str(p))[0]
        trained = models[-1]
        n_trained_lists = len(lists)
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), block, {"restore": True, "save_recs": False}))
        again = run_experiment(str(p))[0]["test_results"][10]
    finally:
        dmf.DMFModel.train_step, dmf.DMF.train, dmf.DMFModel.topk = orig_step, orig_train, orig_topk
    assert res["name"].startswith("DMF_") and "umlp=64-32" in res["name"] and len(res["history"]) == epochs
    E = trained._transactions_per_epoch
    assert E == 6 * trained._data.transactions
    B = E if batch < 1 else batch
    assert len(seen) == epochs * ((E + B - 1) // B)
    ref = ops.MtPointwiseRatioSampler(trained._num_users, trained._num_items, trained._indptr, trained._set_idx,
                                      trained._sampler.set_ratings, trained._sorted_idx, 5, seed=42)
    per_epoch = len(seen) // epochs
    for e in range(epochs):
        ref.epoch()
        want = [t.cpu().numpy() for t in ref.step(E)]
        got = [np.concatenate([s[c] for s in seen[e * per_epoch:(e + 1) * per_epoch]]) for c in range(3)]
        for g_, w in zip(got, want):
            assert np.array_equal(g_, w)
    epoch_sums = [l * (e + 1) for e, l in enumerate(trained._losses)]      # evaluate() gets the epoch sum / (epoch + 1)
    assert np.allclose(epoch_sums, [running[(e + 1) * per_epoch - 1] for e in range(epochs)], rtol=1e-12)
    # the loss falls: the run's first full batches against its last tenth.  Epoch sums are not the measure: at batch
    # 512 or 4 096 the loss settles within the first ~150 steps of the first epoch (with `dot`, outputs below the clip
    # pass no gradient) and later epochs differ only by the noise of the atomics' order in the backward.  An epoch's
    # short last batch is left out: its mean runs over a few samples, normalised among themselves
    run_ = np.array(running).reshape(epochs, per_epoch)
    batch_loss = np.diff(np.concatenate([np.zeros((epochs, 1)), run_], 1), axis=1)
    if E % B:
        batch_loss = batch_loss[:, :-1]
    batch_loss = batch_loss.reshape(-1)
    head, tail = max(1, min(10, batch_loss.size // 10)), max(1, batch_loss.size // 10)
    assert np.isfinite(batch_loss).all()
    assert batch_loss[:head].mean() > batch_loss[-tail:].mean(), (batch_loss[:head], batch_loss[-tail:].mean())
    best = res["test_results"][10]
    for name in ("nDCG", "AUC"):
        assert np.isfinite(best[name]) and again[name] == best[name], name
    assert any(np.array_equal(lists[-1][0], a) and np.array_equal(lists[-1][1], b) for a, b in lists[:n_trained_lists])


def test_c1_rating_metrics_and_bad_widths_refused_before_training(c1_tsv, tmp_path):
    from elliot_b200 import run_experiment
    p = tmp_path / "cfg.yml"
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), {"epochs": 1}, {"save_recs": False}, metrics=("nDCG", "MAE")))
    with pytest.raises(Exception, match="DMF cannot evaluate MAE"):
        run_experiment(str(p))
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), {"epochs": 1, "user_mlp": "(64,20)", "item_mlp": "(64,20)"},
                          {"save_recs": False}))
    with pytest.raises(ValueError, match="multiple of 8"):
        run_experiment(str(p))
