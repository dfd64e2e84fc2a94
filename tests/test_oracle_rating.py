"""CPU tests of MAE, MSE and RMSE and of the SVD++ / FunkSVD restatements: the evaluator's host finishing of a pair pass
against what the unmodified reference Evaluator computed on explicit full lists (tests/golden/rating_metrics_*.npz, minted
by oracle/gen_golden_rating_metrics.py), the oracle's sums on the same lists, the fp64 restatements (oracle/rating_mf.py)
against torch autograd, the evaluator's handling of the names and the refusal of a model without a pair pass."""
import os
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest
import torch

from elliot_b200.dataset import DataSet
from elliot_b200.evaluation import Evaluator
from oracle import rating_mf as oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["MAE", "MSE", "RMSE"]


def frame(a):
    a = np.asarray(a, np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})


def config(thr, metrics=NAMES, cutoffs=(5, 10)):
    return SimpleNamespace(config_test=True, top_k=10,
                           evaluation=SimpleNamespace(simple_metrics=list(metrics), relevance_threshold=thr,
                                                      paired_ttest=False, cutoffs=list(cutoffs)))


def load_cases():
    g = np.load(os.path.join(GOLD, "rating_metrics_cases.npz"))
    out = {c: {k[len(c) + 1:]: g[k] for k in g.files if k.startswith(c + "_")} for c in g["cases"].tolist()}
    c1 = np.load(os.path.join(GOLD, "rating_metrics_c1.npz"))
    out["c1"] = {k: c1[k].astype(np.float64) if k in ("U", "V", "bi", "bu") else c1[k] for k in c1.files}
    out["c1"]["error"] = np.array("")
    return out


def c1_rows():
    from elliot_b200 import synth_c1
    from oracle.gen_golden_rating_metrics import c1_frames
    assert synth_c1.checksum(*synth_c1.rows()) == int(CASES["c1"]["checksum"])
    return c1_frames()[:2]


CASES = load_cases()


def case_data(c, metrics=NAMES):
    g = CASES[c]
    if c == "c1":
        frames = [frame(a) for a in c1_rows()]
    else:
        frames = [frame(g["train"]), frame(g["val"]), frame(g["test"])]
    data = DataSet(config(float(g["thr"]), metrics), tuple(frames))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    return g, data


def full_scores(g):
    return g["U"] @ g["V"].T + g["bi"][None, :] + g["bu"][:, None] + float(g["g"])


def host_pair_scores(g, data, ev):
    """The pair pass on the host: each entry of pair_sets() scored as the user's full list scores it."""
    S = full_scores(g)
    train = data.sp_i_train.tocsr()
    out = {}
    for w, (indptr, items, _) in ev.pair_sets(torch.device("cpu")).items():
        indptr, items = indptr.numpy(), items.numpy().astype(np.int64)
        if items.size == 0:
            out[w] = np.zeros(0, np.float32)
            continue
        rows = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
        s = np.where(items >= 0, S[rows, np.maximum(items, 0)], np.nan)
        in_train = np.asarray(train[rows, np.maximum(items, 0)]).ravel() != 0
        out[w] = np.where((items >= 0) & in_train, -np.inf, s).astype(np.float32)
    return out


def same(a, b):
    return a == b or abs(a - b) <= 1e-12 * abs(b)


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_finish_equals_reference_evaluator(case):
    g, data = case_data(case)
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), score_pass=True)
    scores = host_pair_scores(g, data, ev)
    if str(g["error"]):
        with pytest.raises(ZeroDivisionError):
            ev.eval(({}, {}), pair_scores=scores)
        return
    res = ev.eval(({}, {}), pair_scores=scores)
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, key in enumerate(("val_results", "test_results")):
            for m, name in enumerate(NAMES):
                assert same(res[k][key][name], g["values"][c, s, m]), (case, k, key, name, res[k][key][name])
    if case == "inf":
        assert np.isinf(g["values"][0, 1]).all() and np.isfinite(g["values"][0, 0]).all()


@pytest.mark.parametrize("case", ["thr0", "thr3", "inf"])
def test_oracle_sums_on_full_lists_equal_reference(case):
    """oracle.rating_errors on the explicit full lists, with the test-only items in the denominator."""
    g, data = case_data(case)
    S = full_scores(g)
    train = data.i_train_dict
    from elliot_b200.dataset import eval_csr_of, eval_ratings_of
    indptr, rel, _ = eval_csr_of(data, "test")
    rat = eval_ratings_of(data, "test")
    lists, scores, rels, ratings = {}, {}, {}, {}
    for u in range(data.num_users):
        rest = sorted((i for i in range(data.num_items) if i not in train[u]), key=lambda i: (-S[u, i], i))
        lists[u] = rest + sorted(train[u])
        scores[u] = [S[u, i] for i in rest] + [-np.inf] * len(train[u])
        rels[u], ratings[u] = rel[indptr[u]:indptr[u + 1]].tolist(), rat[indptr[u]:indptr[u + 1]].tolist()
    a, q, n = oracle.rating_errors(lists, scores, rels, ratings)
    assert n == indptr[-1] and (rel < 0).any()
    want = g["values"][0, 1]
    assert same(a / n, want[0]) and same(q / n, want[1]) and same(float(np.sqrt(q / n)), want[2])


def _tables(rng, nu, ni, f, implicit):
    T = {"P": rng.normal(0, 0.3, (nu, f)), "Q": rng.normal(0, 0.3, (ni, f)), "bu": rng.normal(0, 0.1, nu),
         "bi": rng.normal(0, 0.1, ni)}
    if implicit:
        T["Y"] = rng.normal(0, 0.3, (ni, f))
        T["g"] = 0.37
    return T


def _csr(rng, nu, ni):
    rows = [np.sort(rng.choice(ni, size=int(rng.integers(1, ni // 2)), replace=False)) for _ in range(nu)]
    rows[0] = np.array([3])                                             # a one-item row
    return np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64), np.concatenate(rows).astype(np.int64)


def _autograd(T, u, i, y, indptr, indices, implicit):
    t = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in T.items()}
    z = t["P"][u]
    if implicit:
        z = z + torch.stack([t["Y"][indices[indptr[a]:indptr[a + 1]]].mean(0) for a in u])
    out = (z * t["Q"][i]).sum(1) + t["bu"][u] + t["bi"][i] + (t["g"] if implicit else 0.0)
    loss = ((out - torch.tensor(y)) ** 2).mean()
    loss.backward()
    return float(loss.detach()), {k: v.grad.numpy() for k, v in t.items()}


@pytest.mark.parametrize("implicit", [True, False], ids=["svdpp", "funk_svd"])
def test_restatement_matches_autograd(implicit):
    rng = np.random.default_rng(5)
    nu, ni, f, B = 9, 14, 6, 23
    T = _tables(rng, nu, ni, f, implicit)
    indptr, indices = _csr(rng, nu, ni)
    u = rng.integers(0, nu, B); u[:4] = 2                                # repeated users
    i = rng.integers(0, ni, B); y = rng.integers(1, 6, B).astype(np.float64)
    if implicit:
        loss, G, _ = oracle.svdpp_forward_backward(T, u, i, y, indptr, indices)
    else:
        loss, G, _ = oracle.funk_svd_forward_backward(T, u, i, y)
    want_loss, want = _autograd(T, u, i, y, indptr, indices, implicit)
    assert abs(loss - want_loss) <= 1e-12 * abs(want_loss)
    assert sorted(G) == sorted(want)
    for k in G:
        assert np.allclose(G[k], want[k], rtol=1e-12, atol=1e-14), k


@pytest.mark.parametrize("implicit", [True, False], ids=["svdpp", "funk_svd"])
def test_reg_w_and_reg_b_change_nothing(implicit):
    rng = np.random.default_rng(6)
    T = _tables(rng, 7, 11, 4, implicit)
    indptr, indices = _csr(rng, 7, 11)
    u, i, y = rng.integers(0, 7, 16), rng.integers(0, 11, 16), rng.integers(1, 6, 16).astype(np.float64)
    run = (lambda **kw: oracle.svdpp_forward_backward(T, u, i, y, indptr, indices, **kw)) if implicit else \
        (lambda **kw: oracle.funk_svd_forward_backward(T, u, i, y, **kw))
    a, b = run(), run(reg_w=5.0, reg_b=3.0)
    assert a[0] == b[0] and all(np.array_equal(a[1][k], b[1][k]) for k in a[1])


def test_evaluator_accepts_the_names_with_score_pass_only():
    _, data = case_data("thr0")
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), score_pass=True)
    assert ev.needs_pairs and not ev.needs_rank
    with pytest.raises(Exception, match="MAE is not available"):
        Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), score_pass=True)
    with pytest.raises(Exception, match="pair_scores"):
        ev.eval(({}, {}))


@pytest.mark.parametrize("model", ["ItemKNN", "BPRMF", "GMF"])
def test_model_without_pair_pass_refuses_before_training(model, tmp_path):
    import elliot_b200.recommender as R
    if R._bases.HOST != "standalone":
        pytest.skip("the reference's own base classes are bound (the reference package was importable first)")
    _, data = case_data("thr0", metrics=("nDCG", "RMSE"))
    cfg = SimpleNamespace(path_output_rec_weight=str(tmp_path))
    with pytest.raises(Exception, match=f"{model} cannot evaluate RMSE"):
        getattr(R, model)(data, cfg, SimpleNamespace(meta=SimpleNamespace()))
