"""GPU tests of SVD++ and FunkSVD (csrc/rating_mf.cu, recommender/rating_mf.py) and of the MAE / MSE / RMSE pair pass:
the kernels against the fp64 restatements (oracle/rating_mf.py), the rated sampler's distribution, the top-k against the
fp64 bound of oracle/topk_bound.py, the pair pass against the model's own full lists, device against host finishing, and
C1 runs through run_experiment."""
import os
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest
import torch
import yaml

from elliot_b200 import ops, synth_c1
from elliot_b200.dataset import DataSet
from elliot_b200.evaluation import Evaluator
from oracle import rating_mf as oracle
from oracle import tf_models as tfm
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
rel = lambda a, b: np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12)


def _csr(nu, ni, seed, long_user=1):
    """Sorted train rows: row 0 holds one item, row `long_user` most of the catalogue, the others 1 .. 60 items."""
    rs = np.random.RandomState(seed)
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, 60), replace=False)) for _ in range(nu)]
    rows[0] = np.array([5])
    rows[long_user] = np.sort(rs.choice(ni, size=ni - 3, replace=False))
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


def _model(nu, ni, f, implicit, indptr, indices, seed=3):
    from elliot_b200.recommender.rating_mf import RatingMFModel
    m = RatingMFModel(nu, ni, f, 1e-3, seed, torch.from_numpy(indptr).to(DEV), torch.from_numpy(indices).to(DEV), implicit, DEV)
    m.P["bu"][:nu].normal_(0, 0.2); m.P["bi"][:ni].normal_(0, 0.2)
    if implicit:
        m.P["g"][0] = 0.31
    return m


def _host(m, f):
    T = {k: m.P[k][:, :f].double().cpu().numpy() for k in ("P", "Q", "Y") if k in m.P}
    T["bu"] = m.P["bu"][:m.nu].double().cpu().numpy(); T["bi"] = m.P["bi"][:m.ni].double().cpu().numpy()
    if "g" in m.P:
        T["g"] = float(m.P["g"][0])
    return T


@pytest.mark.parametrize("f", [8, 10, 50, 128])
def test_implicit_mean_matches_fp64(f):
    nu, ni = 300, 700
    indptr, indices = _csr(nu, ni, f)
    m = _model(nu, ni, f, True, indptr, indices)
    users = np.r_[np.arange(nu), [1, 1, 0, 7, 7]].astype(np.int32)          # every user, repeats, the 1-item and long rows
    Z = ops.implicit_mean_f32(m.P["P"], m.P["Y"], m.fp, m.indptr, m.indices, users=torch.from_numpy(users).to(DEV))
    T = _host(m, f)
    want = oracle.implicit_means(T["P"], T["Y"], users, indptr, indices)
    got = Z[:, :f].double().cpu().numpy()
    scale = np.abs(T["P"][users]).max(1, keepdims=True) + np.abs(T["Y"]).max()
    assert (np.abs(got - want) <= 1e-6 * scale).all()
    assert not Z[:, m.fp:].any()


@pytest.mark.parametrize("implicit", [True, False], ids=["svdpp", "funk_svd"])
@pytest.mark.parametrize("f", [8, 10, 50, 128])
def test_fused_step_matches_restatement(implicit, f):
    """fp32 kernel vs the fp64 restatement: loss 1e-6, every gradient 1e-5 relative; a full batch with repeated users,
    then a short last batch."""
    nu, ni = 400, 900
    indptr, indices = _csr(nu, ni, 11 + f)
    m = _model(nu, ni, f, implicit, indptr, indices)
    gen = np.random.RandomState(f)
    for B in (2048, 333):
        u = gen.randint(0, nu, B).astype(np.int32); u[:64] = 1; u[64:80] = 0       # the long and the 1-item rows, repeated
        it = gen.randint(0, ni, B).astype(np.int32)
        y = gen.randint(1, 6, B).astype(np.float32)
        T = _host(m, f)
        if implicit:
            loss_ref, G, _ = oracle.svdpp_forward_backward(T, u.astype(np.int64), it, y.astype(np.float64), indptr, indices)
        else:
            loss_ref, G, _ = oracle.funk_svd_forward_backward(T, u.astype(np.int64), it, y.astype(np.float64))
        batch = tuple(torch.from_numpy(a).to(DEV) for a in (u, it, y))
        m._loss.zero_()
        m.grads(batch, m.batch_means(batch[0]) if implicit else None)
        assert abs(m._loss.item() - loss_ref) < 1e-6 * abs(loss_ref)
        for k in ("P", "Q") + (("Y",) if implicit else ()):
            assert rel(m.G[k][:, :f].double().cpu().numpy(), G[k]) < 1e-5, k
            assert not m.G[k][:, f:].any()                                      # padding columns never receive gradient
        assert rel(m.G["bu"][:nu].double().cpu().numpy(), G["bu"]) < 1e-5 and not m.G["bu"][nu:].any()
        assert rel(m.G["bi"][:ni].double().cpu().numpy(), G["bi"]) < 1e-5 and not m.G["bi"][ni:].any()
        if implicit:
            assert abs(m.G["g"][0].item() - G["g"]) < 1e-5 * max(abs(G["g"]), 1e-3) and not m.G["g"][1:].any()
        for k in m.G:
            m.G[k].zero_()


def test_train_step_is_one_keras_adam_step():
    nu, ni, f = 200, 300, 10
    indptr, indices = _csr(nu, ni, 1)
    m = _model(nu, ni, f, True, indptr, indices)
    gen = np.random.RandomState(2)
    u, it = gen.randint(0, nu, 500).astype(np.int32), gen.randint(0, ni, 500).astype(np.int32)
    y = gen.randint(1, 6, 500).astype(np.float32)
    T = _host(m, f)
    _, G, _ = oracle.svdpp_forward_backward(T, u.astype(np.int64), it, y.astype(np.float64), indptr, indices)
    opt = tfm.KerasAdam(1e-3); opt.begin_step()
    want = {k: np.array(v, np.float64) for k, v in T.items()}
    for k in want:
        opt.apply(k, want[k], np.asarray(G[k], np.float64))
    m.train_step(tuple(torch.from_numpy(a).to(DEV) for a in (u, it, y)))
    after = _host(m, f)
    for k in want:
        assert np.abs(np.asarray(after[k]) - want[k]).max() < 2e-6, k
    assert not m.P["bu"][nu:].any() and not m.P["g"][1:].any() and not m.P["Y"][:, f:].any()


def test_rated_sampler_distribution():
    nu, ni = 150, 400
    indptr, indices = _csr(nu, ni, 4)
    ratings = np.random.RandomState(5).randint(1, 6, indices.size).astype(np.float32)
    d = lambda a: torch.from_numpy(a).to(DEV)
    n = 400000
    u, i, r = (t.cpu().numpy() for t in ops.rated_sample_philox(nu, ni, d(indptr), d(indices), d(ratings), n, 42))
    cnt = np.bincount(u, minlength=nu); chi = ((cnt - n / nu) ** 2 / (n / nu)).sum()
    assert abs(chi - (nu - 1)) < 6 * np.sqrt(2 * (nu - 1))                  # users uniform
    pos = np.empty(n, np.int64)
    for x in range(nu):                                                    # items uniform within each row
        sel = u == x
        row = indices[indptr[x]:indptr[x + 1]]
        p = np.searchsorted(row, i[sel])
        assert (row[np.minimum(p, len(row) - 1)] == i[sel]).all()
        pos[sel] = indptr[x] + p
        if len(row) > 1 and sel.sum() > 50 * len(row):
            c = np.bincount(p, minlength=len(row)); e = sel.sum() / len(row)
            assert abs(((c - e) ** 2 / e).sum() - (len(row) - 1)) < 6 * np.sqrt(2 * (len(row) - 1))
    assert np.array_equal(r, ratings[pos])                                 # label = the train rating of (u, i)
    # the stream offset continues the same stream
    u2, i2, _ = ops.rated_sample_philox(nu, ni, d(indptr), d(indices), d(ratings), 1000, 42, first=n - 1000)
    assert np.array_equal(u2.cpu().numpy(), u[-1000:]) and np.array_equal(i2.cpu().numpy(), i[-1000:])


@pytest.mark.parametrize("implicit", [True, False], ids=["svdpp", "funk_svd"])
@pytest.mark.parametrize("k", [10, 50])
def test_topk_against_fp64_with_user_offset(implicit, k):
    nu, ni, f = 500, 1200, 10
    indptr, indices = _csr(nu, ni, 9)
    m = _model(nu, ni, f, implicit, indptr, indices)
    idx, val = m.topk(k, m.indptr, m.indices)
    Z = m.user_vectors()
    if k <= 16:                                                          # the scorer the model lists with
        raw_idx, raw_val, _ = ops.score_topk_tc(Z, m.P["Q"], m.P["bi"], f, k, m.indptr, m.indices, stats=False)
    else:
        raw_idx, raw_val = ops.score_topk(Z, m.P["Q"], m.P["bi"], f, k, m.indptr, m.indices)
    Zh, T = Z[:, :f].double().cpu().numpy(), _host(m, f)
    if implicit:
        assert (np.abs(Zh - oracle.implicit_means(T["P"], T["Y"], np.arange(nu), indptr, indices)) < 1e-5).all()
    filled, total = check_topk_fp64(Zh, T["Q"], T["bi"], f, k, indptr, indices, np.arange(nu), idx.cpu().numpy(),
                                    raw_val.cpu().numpy(), 2.0 ** -24)
    assert total > 0 and filled > 0
    off = T["bu"] + T.get("g", 0.0)
    v = val.double().cpu().numpy()
    assert np.array_equal(idx.cpu().numpy(), raw_idx.cpu().numpy())
    raw = raw_val.double().cpu().numpy()
    fin = np.isfinite(raw)
    assert not fin.all() and np.array_equal(np.isfinite(v), fin)           # the long row runs out of candidates: -inf stays
    assert np.abs(v - (raw + off[:, None]))[fin].max() < 1e-5


def _small_data(thr=3, metrics=("nDCG", "MAE", "MSE", "RMSE")):
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
        simple_metrics=list(metrics), relevance_threshold=thr, paired_ttest=False, cutoffs=[5, 10]))
    return DataSet(cfg, (frame(rows[~test]), frame(te)))


@pytest.mark.parametrize("implicit", [True, False], ids=["svdpp", "funk_svd"])
def test_pair_pass_equals_full_lists_and_reference_formula(implicit):
    from elliot_b200.dataset import train_csr_of
    data = _small_data()
    indptr, _, srt = train_csr_of(data, torch.device(DEV), set_order=False)
    m = _model(data.num_users, data.num_items, 12, implicit, indptr.cpu().numpy(), srt.cpu().numpy())
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), score_pass=True)
    rel_indptr, rel_items, ratings = ev.pair_sets(torch.device(DEV))["test"]
    s = m.pair_scores(rel_indptr, rel_items, indptr, srt).cpu().numpy()
    idx, val = m.topk(data.num_items, indptr, srt)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    rp, ri, rr = rel_indptr.cpu().numpy(), rel_items.cpu().numpy(), ratings.cpu().numpy()
    train = [set(srt[indptr[u]:indptr[u + 1]].cpu().numpy().tolist()) for u in range(data.num_users)]
    lists, scores, rels, rates = {}, {}, {}, {}
    n_inf = 0
    for u in range(data.num_users):
        ok = idx[u] >= 0
        full = dict(zip(idx[u][ok].tolist(), val[u][ok].tolist()))
        for e in range(rp[u], rp[u + 1]):
            it = int(ri[e])
            if it < 0:
                assert np.isnan(s[e])
            elif it in train[u]:
                assert np.isneginf(s[e]); n_inf += 1
            else:
                assert abs(s[e] - full[it]) <= 4e-7 * max(1.0, abs(full[it]))
        tail = sorted(train[u])                                          # the reference's full list ends with them at -inf
        lists[u] = idx[u][ok].tolist() + tail
        scores[u] = val[u][ok].astype(np.float64).tolist() + [-np.inf] * len(tail)
        rels[u], rates[u] = ri[rp[u]:rp[u + 1]].tolist(), rr[rp[u]:rp[u + 1]].tolist()
    assert n_inf == 1 and (ri < 0).sum() == 2
    a, q, n = oracle.rating_errors(lists, scores, rels, rates)
    res = ev.eval(({}, {}), pair_scores={"test": s})[5]["test_results"]
    assert n == rp[-1] and res["MAE"] == a / n == np.inf and res["RMSE"] == np.inf
    # without the train item the sums are finite: the pass against the formula on the lists
    keep = np.isfinite(s) | np.isnan(s)
    d = s.astype(np.float64)[keep & (ri >= 0)] - rr[keep & (ri >= 0)]
    lists2 = {u: [x for x in lists[u] if x not in train[u]] for u in lists}
    scores2 = {u: [v for v in scores[u] if np.isfinite(v)] for u in scores}
    a2, q2, _ = oracle.rating_errors(lists2, scores2, rels, rates)
    assert abs(np.abs(d).sum() - a2) <= 1e-6 * a2 and abs((d * d).sum() - q2) <= 1e-6 * q2


def test_device_finish_equals_host():
    from elliot_b200.dataset import train_csr_of
    data = _small_data(thr=0)
    indptr, _, srt = train_csr_of(data, torch.device(DEV), set_order=False)
    m = _model(data.num_users, data.num_items, 10, True, indptr.cpu().numpy(), srt.cpu().numpy())
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), score_pass=True)
    pairs = {w: m.pair_scores(r[0], r[1], indptr, srt) for w, r in ev.pair_sets(torch.device(DEV)).items()}
    idx, _ = m.topk(10, indptr, srt)
    dev = ev.eval_tensors(idx, pair_scores=pairs)
    host = ev.eval(({}, {}), pair_scores={w: t.cpu().numpy() for w, t in pairs.items()})
    for k in (5, 10):
        for name in ("MAE", "MSE", "RMSE"):
            a, b = dev[k]["test_results"][name], host[k]["test_results"][name]
            assert a == b or abs(a - b) <= 1e-12 * abs(b), (name, a, b)


C1_BLOCK = {"epochs": 5, "batch_size": 512, "factors": 10, "lr": 0.01, "reg_w": 0.1, "reg_b": 0.001, "seed": 7}


@pytest.fixture(scope="module")
def c1_tsv(tmp_path_factory):
    d = tmp_path_factory.mktemp("rating_c1")
    tsv = str(d / "dataset.tsv")
    synth_c1.write_tsv(tsv)
    return tsv


def _c1_yaml(tsv, out, key, meta, device_eval=False):
    block = dict(C1_BLOCK, meta=meta, **({"b200_eval": "device"} if device_eval else {}))
    text = synth_c1.experiment_yaml(tsv, out, key, "", metrics=("nDCG", "MAE", "RMSE", "AUC"), meta=())
    cfg = yaml.safe_load(text)
    cfg["experiment"]["models"][key] = block
    return yaml.safe_dump(cfg)


@pytest.mark.parametrize("key", ["SVDpp", "FunkSVD"])
def test_c1_run_trains_saves_and_restores(c1_tsv, tmp_path, key):
    from elliot_b200 import run_experiment
    from elliot_b200.recommender import rating_mf
    losses = []
    orig = rating_mf._RatingMF.train

    def recording_train(self):                                          # pass-through: keeps the epoch losses
        out = orig(self)
        losses.extend(self._losses)
        return out
    rating_mf._RatingMF.train = recording_train
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"save_weights": True, "save_recs": False}))
        res = run_experiment(str(p))[0]
    finally:
        rating_mf._RatingMF.train = orig
    hist = res["history"]
    assert len(hist) == 5 and res["name"].startswith(key + "_")
    for h in hist:
        assert all(np.isfinite(h[10][m]) for m in ("nDCG", "MAE", "RMSE", "AUC"))
    epoch_sums = [l * (e + 1) for e, l in enumerate(losses)]             # evaluate() gets the epoch sum / (epoch + 1)
    assert epoch_sums[-1] < epoch_sums[0]
    best = res["test_results"][10]
    # the saved weights restore to the same metrics
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"restore": True, "save_recs": False}))
    again = run_experiment(str(p))[0]["test_results"][10]
    for m in ("nDCG", "MAE", "RMSE", "AUC"):
        assert again[m] == best[m], m
    # device evaluation gives the host path's numbers
    p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"restore": True, "save_recs": False}, device_eval=True))
    dev = run_experiment(str(p))[0]["test_results"][10]
    for m in ("nDCG", "MAE", "RMSE", "AUC"):
        assert dev[m] == best[m] or abs(dev[m] - best[m]) <= 1e-12 * abs(best[m]), m
