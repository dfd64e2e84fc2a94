"""CPU tests of AUC and GAUC: the oracle (oracle/auc.py) against what the unmodified reference Evaluator computed on
explicit full lists (tests/golden/auc_cases.npz, minted by oracle/gen_golden_auc.py) and against auc.py / gauc.py
themselves on random lists with ties; the evaluator's finishing function (evaluation.finish_auc) on the counts read off
those lists; the evaluator's handling of the names; and the refusal of a model without a rank pass."""
import os
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest

from elliot_b200.dataset import DataSet, eval_csr_of
from elliot_b200.evaluation import Evaluator, finish_auc
from oracle import auc as oracle
from oracle import ref_stubs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def frame(a):
    a = np.asarray(a, np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})


def config(thr, metrics=("AUC", "GAUC"), cutoffs=(5, 10)):
    return SimpleNamespace(config_test=True, top_k=10,
                           evaluation=SimpleNamespace(simple_metrics=list(metrics), relevance_threshold=thr,
                                                      paired_ttest=False, cutoffs=list(cutoffs)))


def cases():
    g = np.load(os.path.join(GOLD, "auc_cases.npz"))
    return {c: {k[len(c) + 1:]: g[k] for k in g.files if k.startswith(c + "_")} for c in g["cases"].tolist()}


CASES = cases()


def case_data(c, metrics=("AUC", "GAUC")):
    g = CASES[c]
    data = DataSet(config(float(g["thr"]), metrics), (frame(g["train"]), frame(g["val"]), frame(g["test"])))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    return g, data


def split_inputs(g, data, which):
    """{private user: full list}, {private user: relevant private items (-1: test-only)}, {private user: |train_u|}."""
    lp, li = g["list_indptr"], g["list_items"]
    lists = {u: li[lp[u]:lp[u + 1]].tolist() for u in range(data.num_users)}
    indptr, rel, _ = eval_csr_of(data, which)
    rels = {u: rel[indptr[u]:indptr[u + 1]].tolist() for u in range(data.num_users)}
    n_train = np.diff(data.sp_i_train.tocsr().indptr)
    return lists, rels, dict(enumerate(n_train.tolist())), indptr, n_train


def close(a, b):
    return (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-12 * max(1.0, abs(b))


@pytest.mark.parametrize("model", ["ItemKNN", "EASER", "NeuMF", "MultiVAE"])
def test_model_without_rank_pass_refuses_before_training(model, tmp_path):
    import elliot_b200.recommender as R
    if R._bases.HOST != "standalone":
        pytest.skip("the reference's own base classes are bound (the reference package was importable first)")
    _, data = case_data("ties", metrics=("nDCG", "AUC"))
    cfg = SimpleNamespace(path_output_rec_weight=str(tmp_path))
    with pytest.raises(Exception, match=f"{model} cannot evaluate AUC"):
        getattr(R, model)(data, cfg, SimpleNamespace(meta=SimpleNamespace()))


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_and_finish_equal_reference_evaluator(case):
    g, data = case_data(case)
    for s, which in enumerate(("val", "test")):
        lists, rels, n_train, indptr, n_train_arr = split_inputs(g, data, which)
        counts = [oracle.rank_counts(lists[u], rels[u]) for u in range(data.num_users)]
        n_pos = [c[0] for c in counts]
        sum_c = [c[1] for c in counts]
        if str(g["error"]):                            # the reference raised on the test split (user 7 has no val rows)
            if which == "val":
                continue
            with pytest.raises(ZeroDivisionError):
                oracle.auc_gauc(lists, rels, data.num_items, n_train)
            with pytest.raises(ZeroDivisionError):
                finish_auc(n_pos, sum_c, np.diff(indptr), n_train_arr, data.num_items, ["AUC", "GAUC"])
            continue
        want = g["values"][0, s]
        assert np.array_equal(g["values"][0], g["values"][1], equal_nan=True)          # the same at every cutoff
        got = oracle.auc_gauc(lists, rels, data.num_items, n_train)
        fin = finish_auc(n_pos, sum_c, np.diff(indptr), n_train_arr, data.num_items, ["AUC", "GAUC"])
        for m, w, o in zip(("AUC", "GAUC"), want, got):
            assert close(o, w), (case, which, m, o, w)
            assert close(fin[m], w), (case, which, m, fin[m], w)


def test_big_case_exceeds_one_rank_chunk():
    g, data = case_data("big")
    indptr = eval_csr_of(data, "test")[0]
    assert np.diff(indptr).max() > 1024


@pytest.mark.skipif(not ref_stubs.available(), reason="the reference project is not present")
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_reproduces_reference_metric_classes_on_random_lists(seed):
    ref_stubs.install()
    auc_mod = ref_stubs.load(os.path.join(ref_stubs.REF, "elliot/evaluation/metrics/accuracy/AUC/auc.py"), "ref_auc")
    gauc_mod = ref_stubs.load(os.path.join(ref_stubs.REF, "elliot/evaluation/metrics/accuracy/AUC/gauc.py"), "ref_gauc")
    rng = np.random.default_rng(seed)
    n_items, n_users = 60, 40
    lists, rels, train, recs = {}, {}, {}, {}
    for u in range(n_users):
        tr = rng.choice(n_items, size=int(rng.integers(0, 20)), replace=False)
        rest = np.setdiff1d(np.arange(n_items), tr)
        scores = rng.integers(-2, 3, size=rest.size).astype(float)         # ties
        order = np.lexsort((rest, -scores))
        lists[u] = rest[order].tolist()
        pool = np.r_[rest, [n_items + 1, n_items + 2]]                     # two ids outside the catalogue
        rels[u] = rng.choice(pool, size=int(rng.integers(0, 12)), replace=False).tolist() if u % 7 else []
        train[u] = {int(i): 1 for i in tr}
        recs[u] = [(i, float(s)) for i, s in zip(rest[order].tolist(), scores[order].tolist())]
    rel = SimpleNamespace(binary_relevance=SimpleNamespace(get_user_rel=lambda u: rels.get(u, [])))
    objs = SimpleNamespace(cutoff=10, relevance=rel, num_items=n_items, data=SimpleNamespace(train_dict=train))
    want_auc = auc_mod.AUC(recs, None, None, objs).eval()
    want_gauc = gauc_mod.GAUC(recs, None, None, objs).eval()
    got = oracle.auc_gauc(lists, rels, n_items, {u: len(t) for u, t in train.items()})
    assert close(got[0], want_auc) and close(got[1], want_gauc)
    counts = [oracle.rank_counts(lists[u], rels[u]) for u in range(n_users)]
    fin = finish_auc([c[0] for c in counts], [c[1] for c in counts], [len(rels[u]) for u in range(n_users)],
                     [len(train[u]) for u in range(n_users)], n_items, ["GAUC", "AUC"])
    assert list(fin) == ["GAUC", "AUC"]
    assert close(fin["AUC"], want_auc) and close(fin["GAUC"], want_gauc)


def test_evaluator_takes_the_names_and_asks_for_top_k_lists():
    g, data = case_data("ties", metrics=("nDCG", "auc", "GAUC"))
    with pytest.raises(Exception, match="not available.*rank pass"):          # no source of rank counts
        Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), rank_pass=True)
    assert ev.needs_rank and ev.get_needed_recommendations() == 10
    recs = {u: [] for u in data.users}
    with pytest.raises(Exception, match="rank pass"):
        ev.eval((recs, recs))
    _, data2 = case_data("ties", metrics=("nDCG", "HR"))
    assert not Evaluator(data2, SimpleNamespace(meta=SimpleNamespace()), rank_pass=True).needs_rank


def test_evaluator_copies_the_rank_values_into_every_cutoff():
    g, data = case_data("thr3", metrics=("HR", "GAUC", "AUC"))
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()), rank_pass=True)
    counts = {}
    for which in ("val", "test"):
        lists, rels, *_ = split_inputs(g, data, which)
        c = [oracle.rank_counts(lists[u], rels[u]) for u in range(data.num_users)]
        counts[which] = (np.array([x[0] for x in c]), np.array([x[1] for x in c]))
    lp, li = g["list_indptr"], g["list_items"]
    recs = {data.users[u]: [(data.items[i], 0.0) for i in li[lp[u]:lp[u + 1]][:10]] for u in range(data.num_users)}
    res = ev.eval((recs, recs), rank_counts=counts)
    for c, k in enumerate((5, 10)):
        for s, split in enumerate(("val_results", "test_results")):
            assert list(res[k][split]) == ["HR", "GAUC", "AUC"]
            assert close(res[k][split]["AUC"], g["values"][c, s, 0]) and close(res[k][split]["GAUC"], g["values"][c, s, 1])
