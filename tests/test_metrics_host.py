"""CPU tests of the evaluator's 19 list metrics beyond nDCG / HR / Precision / Recall (elliot_b200/evaluation.py):
the host mirror against what the unmodified reference Evaluator computed on the same lists (tests/golden/metrics_*.npz,
minted by oracle/gen_golden_metrics.py), the static tables against the reference's Popularity and per-user loops, the
names that stay out of scope, ZeroDivisionError parity, and a new metric as validation metric and early-stopping
monitor."""
import os
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest

from elliot_b200.dataset import DataSet, eval_csr_of, eval_users_of
from elliot_b200.evaluation import PER_USER, Evaluator, host_metric_sums

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
INTEGER = ("ItemCoverage", "UserCoverage", "UserCoverageAtN")


def frame(a):
    a = np.asarray(a, np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})


def config(top_k, cutoffs, thr, metrics):
    return SimpleNamespace(config_test=False, top_k=top_k,
                           evaluation=SimpleNamespace(simple_metrics=list(metrics), relevance_threshold=thr,
                                                      paired_ttest=False, cutoffs=list(cutoffs)))


def cases():
    g = np.load(os.path.join(GOLD, "metrics_cases.npz"))
    return {c: {k[len(c) + 1:]: g[k] for k in g.files if k.startswith(c + "_")} for c in g["cases"].tolist()}


CASES = cases()


def case_data(c, metrics=None):
    """The mirror's DataSet and Evaluator on a golden case; its private ids must be the reference's."""
    g = CASES[c]
    data = DataSet(config(int(g["top_k"]), g["cutoffs"].tolist(), float(g["thr"]), metrics or g["metrics"].tolist()),
                   (frame(g["train"]), frame(g["val"]), frame(g["test"])))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    return g, data, Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))


def as_recs(data, idx):
    """{public user: [(public item, score)]} of a private-id array (-1 ends a list)."""
    out = {}
    for pu, row in enumerate(idx):
        row = row[:np.argmax(row < 0)] if (row < 0).any() else row
        out[data.users[pu]] = [(data.items[i], float(len(row) - q)) for q, i in enumerate(row.tolist())]
    return out


def assert_close(got, want, what):
    for m, w in want.items():
        if m in INTEGER:
            assert got[m] == w and isinstance(got[m], int), (*what, m, got[m], w)
        else:
            assert abs(got[m] - w) <= 1e-12 * max(1.0, abs(w)), (*what, m, got[m], w)


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_mirror_equals_reference_evaluator(case):
    g, data, ev = case_data(case)
    names = g["metrics"].tolist()
    recs = as_recs(data, g["rec_idx"])
    res = ev.eval((recs, recs))
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, split in enumerate(("val_results", "test_results")):
            assert list(res[k][split]) == names                           # config order
            assert_close(res[k][split], dict(zip(names, g["values"][c, s].tolist())), (case, k, split))


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_per_user_values_equal_reference(case):
    g, data, ev = case_data(case)
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, which in enumerate(("val", "test")):
            _, per = host_metric_sums(ev._tables(which), ev._sets[which], np.arange(data.num_users), g["rec_idx"], k,
                                      per_user=True)
            want = g["per_user"][c, s].T
            asked = [j for j, m in enumerate(PER_USER) if m in g["metrics"].tolist()]
            np.testing.assert_array_equal(np.isnan(per[:, asked]), np.isnan(want[:, asked]))
            np.testing.assert_allclose(per[:, asked], want[:, asked], rtol=1e-12, atol=1e-15)


def test_host_mirror_equals_reference_at_c1():
    from elliot_b200 import synth_c1
    from elliot_b200.run import _read, split_random_subsampling
    g = np.load(os.path.join(GOLD, "metrics_c1.npz"))
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        tsv = os.path.join(tmp, "dataset.tsv")
        assert synth_c1.write_tsv(tsv) == int(g["checksum"])
        df = _read(tsv, False)
    (train, test), = split_random_subsampling(df, 0.2, 42)
    names = g["metrics"].tolist()
    data = DataSet(config(int(g["top_k"]), g["cutoffs"].tolist(), 0, names), (train, test))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    recs = as_recs(data, g["rec_idx"])
    res = ev.eval((recs, recs))
    for c, k in enumerate(g["cutoffs"].tolist()):
        assert_close(res[k]["test_results"], dict(zip(names, g["values"][c].tolist())), ("c1", k))


@pytest.mark.parametrize("case", sorted(CASES))
def test_static_tables_equal_reference_popularity_and_per_user_loops(case):
    g, data, ev = case_data(case)
    assert set(np.flatnonzero(ev._tables("test").long_tail == 0).tolist()) == set(g["short_head"].tolist())
    train = data.i_train_dict
    short_head = set(g["short_head"].tolist())
    long_tail = set(range(data.num_items)) - short_head
    pop = [sum(i in train[u] for u in train) for i in range(data.num_items)]
    for which in ("val", "test"):
        tab = ev._tables(which)
        assert tab.pop.tolist() == pop
        d = data.test_dict if which == "test" else data.val_dict
        thr = data.config.evaluation.relevance_threshold
        for pu, u in enumerate(data.users):                              # pop_reo.py / pop_rsp.py / lauc.py, per user
            rel = {data.public_items.get(i, -1) for i, r in d[u].items() if r >= thr} - {-1}
            tr = set(train[pu])
            want = [bool(d[u]), len(tr), len((short_head & rel) - tr), len((long_tail & rel) - tr),
                    len(short_head - tr), len(long_tail - tr)]
            assert tab.user_info[pu].tolist() == want, (which, pu)
        n_users = data.num_users
        np.testing.assert_array_equal(tab.nov[:, 0], 1 - np.array(pop) / n_users)
        assert np.array_equal(eval_users_of(data, which), np.array([bool(d[u]) for u in data.users]))


def test_has_test_rows_mask_separates_from_relevant_users():
    g, data, ev = case_data("b")                                        # threshold 3
    rows = eval_users_of(data, "test")
    indptr = eval_csr_of(data, "test")[0]
    rel = np.diff(indptr) > 0
    assert np.all(rows[rel]) and (rows & ~rel).any() and (~rows).any()


@pytest.mark.parametrize("name", ["AUC", "GAUC", "MAE", "MSE", "RMSE", "DSC", "ExtendedF1", "ExtendedEPC", "SRecall",
                                  "BiasDisparityBD", "UserMADrating", "REO", "RSP", "NumRetrived"])
def test_out_of_scope_names_raise(name):
    with pytest.raises(Exception, match="not available"):
        case_data("a", metrics=["nDCG", name])


def test_empty_list_under_arp_raises_like_the_reference():
    g, data, ev = case_data("c", metrics=["HR", "ARP"])                 # case c has one empty list of a user with test rows
    recs = as_recs(data, g["rec_idx"])
    with pytest.raises(ZeroDivisionError):
        ev.eval((recs, recs))
    _, _, ev = case_data("c", metrics=["HR", "ACLT", "Gini"])
    ev.eval((recs, recs))


def test_four_metric_results_unchanged_by_the_new_ones():
    g, data, ev = case_data("a", metrics=["nDCG", "HR", "Precision", "Recall"])
    _, _, ev2 = case_data("a", metrics=["MAP", "nDCG", "Gini", "HR", "Precision", "Recall"])
    recs = as_recs(data, g["rec_idx"])
    a, b = ev.eval((recs, recs)), ev2.eval((recs, recs))
    for k in a:
        for m in ("nDCG", "HR", "Precision", "Recall"):
            assert a[k]["test_results"][m] == b[k]["test_results"][m]
        assert list(b[k]["test_results"]) == ["MAP", "nDCG", "Gini", "HR", "Precision", "Recall"]


def test_new_metric_as_validation_metric_and_early_stopping_monitor():
    from elliot_b200.recommender.base_recommender_model import BaseRecommenderModel
    from elliot_b200.recommender.recommender_utils_mixin import RecMixin

    class M(RecMixin, BaseRecommenderModel):
        train = get_recommendations = get_params = lambda self, *a: None

    g, data, ev = case_data("a")
    params = SimpleNamespace(meta=SimpleNamespace(validation_metric="MAP@10"), epochs=5,
                             early_stopping={"monitor": "Gini@5", "patience": 1})
    m = M(data, SimpleNamespace(), params)
    assert (m._validation_metric, m._validation_k) == ("MAP", 10)
    idx = g["rec_idx"].copy()
    for shrink in (0, 3, 6):                                             # fewer listed items each round
        if shrink:
            idx[:, -shrink:] = -1
        recs = as_recs(data, idx)
        m._results.append(ev.eval((recs, recs)))
        m._losses.append(0.0)
    maps = [r[10]["val_results"]["MAP"] for r in m._results]
    assert m.get_best_arg() == int(np.argmax(maps))
    ginis = [r[5]["val_results"]["Gini"] for r in m._results]
    assert m._early_stopping.stop(m._losses, m._results) == (ginis[1] > ginis[2])   # patience 1: the newest got worse
