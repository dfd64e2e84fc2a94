"""GPU tests of the AUC / GAUC rank pass (eb_score_rank_*, ops.score_rank): the per-positive counts against the full
lists ops.score_topk(k=n_items) gives for the same tables, bit-identical reruns, the reference's AUC / GAUC on the
golden cases (tests/golden/auc_cases.npz), and run_experiment: the C1 BPRMF run against the reference's own run with
AUC / GAUC (tests/golden/auc_c1.npz), unchanged lists and metrics when AUC / GAUC are added, every model with a rank
pass under both evaluation paths, and the refusal of a model without one."""
import os

import numpy as np
import pytest
import torch
import yaml

from elliot_b200 import ops, synth_c1
from elliot_b200.evaluation import finish_auc
from oracle import auc as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def to_dev(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)


def random_tables(rng, n_users, n_items, d, dtype, bias=True, specials=False):
    U = rng.standard_normal((n_users, d))
    V = rng.standard_normal((n_items, d))
    b = rng.standard_normal(n_items) if bias else None
    if specials:                                           # items never listed: -inf and NaN scores
        b[rng.choice(n_items, 5, replace=False)] = -np.inf
        b[rng.choice(n_items, 5, replace=False)] = np.nan
    t = lambda a: None if a is None else to_dev(a, dtype)
    return t(U), t(V), t(b)


def random_csrs(rng, n_users, n_items, big_user=None):
    """Train CSR (sorted, some rows empty) and an item-sorted relevant CSR with -1 entries, disjoint from train."""
    tp, ti, rp, ri = [0], [], [0], []
    for u in range(n_users):
        n_tr = 0 if u % 5 == 0 else int(rng.integers(1, 40))
        n_rel = int(rng.integers(0, 12)) if u != big_user else 1500
        items = rng.choice(n_items, size=min(n_items, n_tr + n_rel), replace=False)
        tr, rel = np.sort(items[:n_tr]), items[n_tr:].tolist()
        rel += [-1] * int(u % 3 == 1)                       # an item outside the catalogue
        ti += tr.tolist(); tp.append(len(ti))
        ri += sorted(rel); rp.append(len(ri))
    return (to_dev(tp, torch.int64), to_dev(ti, torch.int32)), (to_dev(rp, torch.int64), to_dev(ri, torch.int32))


def counts_from_full_lists(idx, users, rel_indptr, rel_items):
    """Per relevant-CSR entry: the non-relevant entries ahead of it in the user's full list, -1 when not listed."""
    idx, rp, ri = idx.cpu().numpy(), rel_indptr.cpu().numpy(), rel_items.cpu().numpy()
    c = np.full(ri.size, -1, np.int64)
    for q, u in enumerate(users):
        rel = {int(i): e for e, i in enumerate(ri[rp[u]:rp[u + 1]], rp[u])}
        ahead = 0
        for it in idx[q]:
            if it < 0:
                break
            if int(it) in rel:
                c[rel[int(it)]] = ahead
            else:
                ahead += 1
    return c


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("variant", ["all", "subset", "no_bias", "big", "specials"])
def test_counts_equal_full_score_topk_lists(dtype, variant):
    rng = np.random.default_rng(7)
    n_users, n_items, d = 48, 1800 if variant == "big" else 700, 40
    U, V, b = random_tables(rng, n_users, n_items, d, dtype, bias=variant != "no_bias", specials=variant == "specials")
    (mp, mi), (rp, ri) = random_csrs(rng, n_users, n_items, big_user=3 if variant == "big" else None)
    users = to_dev(rng.permutation(n_users)[:17], torch.int32) if variant == "subset" else None
    ulist = users.cpu().numpy() if users is not None else np.arange(n_users)
    idx, _ = ops.score_topk(U, V, b, d, n_items, mp, mi, users=users)
    want = counts_from_full_lists(idx, ulist, rp, ri)
    n_pos, sum_c, c = ops.score_rank(U, V, b, d, rp, ri, mp, mi, users=users, per_positive=True)
    c = c.cpu().numpy()
    np.testing.assert_array_equal(c, want)
    rpn = rp.cpu().numpy()
    for q, u in enumerate(ulist):
        cu = want[rpn[u]:rpn[u + 1]]
        assert n_pos[q].item() == (cu >= 0).sum() and sum_c[q].item() == cu[cu >= 0].sum(), (q, u)
    if variant == "big":
        assert (want[rpn[3]:rpn[4]] >= 0).sum() > 1024
    n2, s2, c2 = ops.score_rank(U, V, b, d, rp, ri, mp, mi, users=users, per_positive=True)   # reruns: same bits
    assert torch.equal(n2, n_pos) and torch.equal(s2, sum_c) and np.array_equal(c2.cpu().numpy(), c)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_catalogue_beyond_any_bitmap(dtype):
    """70 000 items, integer tables (every score exact in any order): the counts against a host sort."""
    rng = np.random.default_rng(3)
    n_users, n_items, d = 12, 70_000, 8
    U = rng.integers(-3, 4, size=(n_users, d)).astype(np.float64)
    V = rng.integers(-3, 4, size=(n_items, d)).astype(np.float64)
    b = rng.integers(-2, 3, size=n_items).astype(np.float64)
    (mp, mi), (rp, ri) = random_csrs(rng, n_users, n_items)
    _, _, c = ops.score_rank(to_dev(U, dtype), to_dev(V, dtype), to_dev(b, dtype), d, rp, ri, mp, mi, per_positive=True)
    S = U @ V.T + b
    mpn, min_, rpn, rin = (t.cpu().numpy() for t in (mp, mi, rp, ri))
    want = np.full(rin.size, -1, np.int64)
    for u in range(n_users):
        keep = np.ones(n_items, bool)
        keep[min_[mpn[u]:mpn[u + 1]]] = False
        items = np.flatnonzero(keep)
        lst = items[np.lexsort((items, -S[u, items]))]
        rel = rin[rpn[u]:rpn[u + 1]].tolist()
        _, _, cs = oracle.rank_counts(lst.tolist(), rel)
        pos = [e for e in range(rpn[u], rpn[u + 1]) if rin[e] >= 0 and keep[rin[e]]]
        pos.sort(key=lambda e: (-S[u, rin[e]], rin[e]))
        want[pos] = cs
    np.testing.assert_array_equal(c.cpu().numpy(), want)


# ---------------------------------------------------------------- golden cases
def frame(a):
    import pandas as pd
    a = np.asarray(a, np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})


def gold_cases():
    g = np.load(os.path.join(GOLD, "auc_cases.npz"))
    return {c: {k[len(c) + 1:]: g[k] for k in g.files if k.startswith(c + "_")} for c in g["cases"].tolist()}


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", ["big", "no_positive", "thr3", "ties", "zero_neg"])
def test_golden_cases_give_the_reference_values(case, dtype):
    from types import SimpleNamespace
    from elliot_b200.dataset import DataSet, train_csr_of
    from elliot_b200.evaluation import Evaluator
    g = gold_cases()[case]
    cfg = SimpleNamespace(config_test=True, top_k=10, evaluation=SimpleNamespace(
        simple_metrics=["AUC", "GAUC"], relevance_threshold=float(g["thr"]), paired_ttest=False, cutoffs=[5, 10]))
    data = DataSet(cfg, tuple(frame(g[k]) for k in ("train", "val", "test")))
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), rank_pass=True)
    mp, _, mi = train_csr_of(data, DEV, set_order=False)
    U, V, b = (to_dev(g[k], dtype) for k in ("U", "V", "bias"))
    counts = {w: tuple(t.cpu().numpy() for t in ops.score_rank(U, V, b, U.shape[1], *rel, mp, mi))
              for w, rel in ev.rank_sets(DEV).items()}
    n_train = np.diff(data.sp_i_train.tocsr().indptr)
    for s, which in enumerate(("val", "test")):
        n_rel = np.diff(ev._sets[which][0])
        if str(g["error"]) and which == "test":
            with pytest.raises(ZeroDivisionError):
                finish_auc(*counts[which], n_rel, n_train, data.num_items, ["AUC", "GAUC"])
            continue
        if str(g["error"]):
            continue
        got = finish_auc(*counts[which], n_rel, n_train, data.num_items, ["AUC", "GAUC"])
        for m, w in zip(("AUC", "GAUC"), g["values"][0, s]):
            assert (np.isnan(w) and np.isnan(got[m])) or abs(got[m] - w) <= 1e-12, (case, which, m, got[m], w)


# ---------------------------------------------------------------- run_experiment
def run_yaml(out, text):
    from elliot_b200 import run_experiment
    os.makedirs(out, exist_ok=True)
    (out / "cfg.yml").write_text(text)
    return run_experiment(str(out / "cfg.yml"))[0]


@pytest.fixture(scope="module")
def c1(tmp_path_factory):
    g = dict(np.load(os.path.join(GOLD, "auc_c1.npz")))
    d = tmp_path_factory.mktemp("auc_c1")
    tsv = str(d / "dataset.tsv")
    assert synth_c1.write_tsv(tsv) == int(g["checksum"]), "this numpy draws a different synthetic file than the golden's"
    return g, d, tsv


def c1_yaml(tsv, out, metrics, save_recs=False):
    return synth_c1.yaml_text(tsv, str(out), "BPRMF", 1, 64, save_recs=save_recs, metrics=metrics)


def test_c1_bprmf_run_gives_the_reference_auc(c1):
    g, d, tsv = c1
    names = g["metrics"].tolist()
    res = run_yaml(d / "exact", c1_yaml(tsv, d / "exact", names))
    got = res["test_results"][10]
    diffs = {m: abs(got[m] - w) for m, w in zip(names, g["values"].tolist())}
    print("C1 |ours - reference|:", diffs)
    for m, w in zip(names, g["values"].tolist()):
        assert diffs[m] <= (1e-6 if m in ("AUC", "GAUC") else 1e-4), (m, got[m], w)


def test_c1_lists_and_other_metrics_unchanged_by_auc(c1):
    g, d, tsv = c1
    base = ["nDCG", "HR", "Precision", "Recall"]
    a = run_yaml(d / "plain", c1_yaml(tsv, d / "plain", base, save_recs=True))
    b = run_yaml(d / "auc", c1_yaml(tsv, d / "auc", ["AUC"] + base + ["GAUC"], save_recs=True))
    for m in base:
        assert a["test_results"][10][m] == b["test_results"][10][m], m
    fa, fb = (sorted(os.listdir(p / "recs")) for p in (d / "plain", d / "auc"))
    assert fa == fb and fa
    for f in fa:
        assert (d / "plain" / "recs" / f).read_bytes() == (d / "auc" / "recs" / f).read_bytes(), f


SMALL_BLOCKS = {
    "BPRMF": {"epochs": 1, "factors": 8},
    "BPRMF_hogwild": {"epochs": 1, "factors": 8, "b200_mode": "hogwild", "b200_batch": 2048},
    "BPRMF_batch": {"epochs": 1, "factors": 8, "batch_size": 256},
    "MF2020": {"epochs": 1, "factors": 8},
    "GMF": {"epochs": 1, "mf_factors": 8, "batch_size": 256},
    "iALS": {"epochs": 1, "factors": 8},
    "WRMF": {"epochs": 1, "factors": 8},
    "PureSVD": {"factors": 8},
    "NonNegMF": {"epochs": 1, "factors": 8, "batch_size": 256},
}


def small_yaml(tmp, key, block, device_eval):
    g = gold_cases()["thr3"]
    for name in ("train", "val", "test"):
        with open(tmp / f"{name}.tsv", "w") as f:
            f.writelines(f"{int(u)}\t{int(i)}\t{r}\n" for u, i, r in g[name])
    block = dict(block, meta={"save_recs": False}, b200_eval="device" if device_eval else "host")
    cfg = {"experiment": {"dataset": "auc_small", "data_config": {"strategy": "fixed", "train_path": "train.tsv",
                                                                 "validation_path": "val.tsv", "test_path": "test.tsv"},
                          "top_k": 10, "evaluation": {"simple_metrics": ["HR", "AUC", "GAUC"], "cutoffs": [5, 10],
                                                      "relevance_threshold": 3},
                          "path_output_rec_result": str(tmp / "recs"), "path_output_rec_weight": str(tmp / "w"),
                          "path_output_rec_performance": str(tmp / "perf"), "models": {key.split("_hogwild")[0]: block}}}
    return yaml.safe_dump(cfg)


@pytest.mark.parametrize("device_eval", [False, True])
@pytest.mark.parametrize("key", sorted(SMALL_BLOCKS))
def test_every_ranking_model_equals_the_oracle_on_its_full_lists(tmp_path, key, device_eval, monkeypatch):
    from elliot_b200.recommender.recommender_utils_mixin import RecMixin
    seen = []
    orig = RecMixin.evaluate

    def recording(self, *a, **k):                      # pass-through: keeps the model to read its tables afterwards
        seen.append(self)
        return orig(self, *a, **k)
    monkeypatch.setattr(RecMixin, "evaluate", recording)
    res = run_yaml(tmp_path, small_yaml(tmp_path, key, SMALL_BLOCKS[key], device_eval))
    model = seen[-1]
    data, ev = model._data, model.evaluator
    idx, _ = model._model.get_recs_topk(data.num_items, model._indptr, model._sorted_idx) if key == "GMF" else \
        ops.score_topk(*model_tables(model), data.num_items, model._indptr, model._sorted_idx)
    idx = idx.cpu().numpy()
    lists = {u: [int(i) for i in idx[u] if i >= 0] for u in range(data.num_users)}
    n_train = dict(enumerate(np.diff(data.sp_i_train.tocsr().indptr).tolist()))
    for which, split in (("val", "val_results"), ("test", "test_results")):
        indptr, rel, _ = ev._sets[which]
        rels = {u: rel[indptr[u]:indptr[u + 1]].tolist() for u in range(data.num_users)}
        want = oracle.auc_gauc(lists, rels, data.num_items, n_train)
        for k in (5, 10):
            got = res[split][k]
            assert abs(got["AUC"] - want[0]) <= 1e-12 and abs(got["GAUC"] - want[1]) <= 1e-12, (which, k, got, want)


def model_tables(model):
    """(U, V, bias, d) of the table scoring the lists the model's topk selects from."""
    m = model._model
    name = type(model).__name__
    if name == "BPRMF":
        return m.U, m.V, m.b, m._factors
    if name == "BPRMF_batch":
        return m.Gu, m.Gi, m.Bi[:m._num_items], m._factors
    if name == "MF2020":
        return m.U, m.V, m.ib, m._factors
    if name in ("iALS", "WRMF"):
        return m.X, m.Y, None, m.d
    if name == "PureSVD":
        return m.user_vec, m.item_vec, None, m.d
    if name == "NonNegMF":
        return m.P, m.Q, m.bi, m.F
    raise AssertionError(name)


def test_model_without_rank_pass_refuses_before_training(tmp_path):
    text = small_yaml(tmp_path, "ItemKNN", {"neighbors": 20, "similarity": "cosine"}, False)
    with pytest.raises(Exception, match="ItemKNN cannot evaluate AUC/GAUC"):
        run_yaml(tmp_path, text)
    assert not os.path.exists(tmp_path / "w") or not os.listdir(tmp_path / "w")
