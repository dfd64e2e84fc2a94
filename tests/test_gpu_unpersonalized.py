"""MostPop and Random on the GPU: the kernels' lists against the reference's dicts (tests/golden/unpersonalized_cases.npz)
and the oracle, under users= subsets too; the stream continuing across calls; run_experiment on the C1 file with both
models (rec-file lines and metrics against the reference's run, host and device evaluation); the device metric kernel
on lists with duplicate items; and the AUC refusal."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

import c1_harness as c1h
import unpersonalized_cases as uc
from c1_harness import DEV, to_dev
from elliot_b200 import ops, synth_c1
from elliot_b200.evaluation import Evaluator
from elliot_b200.recommender.unpersonalized import MostPopLists, RandomLists
from oracle import unpersonalized as oun

pytestmark = pytest.mark.gpu


def _model(cls, data, **kw):
    """A model instance with only the fields its list methods read."""
    m = object.__new__(cls)
    m._data, m._negative_sampling = data, False
    m._lists = (MostPopLists(data, DEV) if cls.__name__ == "MostPop" else RandomLists(data, kw["seed"], DEV))
    if cls.__name__ == "MostPop":
        m._lists.initialize()
    return m


def test_mostpop_lists_equal_the_reference():
    from elliot_b200.recommender import MostPop
    g = uc.case("mostpop")
    data = uc.data_of(g)
    m = _model(MostPop, data)
    k = int(g["k"])
    assert uc.same_dict(m.get_single_recommendation(None, k), uc.golden_dict(g))
    assert not m.lists_are_tensors(k) and m.lists_are_tensors(1)
    idx, val, skipped = ops.mostpop_topk(m._lists.order, m._lists.pop, k, m._lists.indptr, m._lists.train)
    rows, pop, skip = oun.mostpop(*uc.train_csr(data), data.num_items, k)
    assert np.array_equal(idx.cpu().numpy(), rows) and np.array_equal(val.cpu().numpy(), pop)
    assert int(skipped) == skip.sum() == 2
    users = np.array([20, 3, 5, 0, 11, 3], np.int32)                # skipped, colliding, repeated, one short
    si, sv, ss = ops.mostpop_topk(m._lists.order, m._lists.pop, k, m._lists.indptr, m._lists.train,
                                  users=to_dev(users))
    assert np.array_equal(si.cpu().numpy(), rows[users]) and np.array_equal(sv.cpu().numpy(), pop[users])
    assert int(ss) == 2
    bi, _, _ = ops.mostpop_topk(m._lists.order, m._lists.pop, k, m._lists.indptr, m._lists.train, user_begin=17, n_sel=9)
    assert np.array_equal(bi.cpu().numpy(), rows[17:26])


def test_item_pop_counts_train_users():
    g = np.random.default_rng(3)
    n_items = 5000
    M = g.random((700, n_items)) < g.random(n_items) ** 4
    indices = np.nonzero(M)[1].astype(np.int32)
    pop = ops.item_pop(to_dev(indices), n_items).cpu().numpy()
    assert np.array_equal(pop, M.sum(0))


@pytest.mark.parametrize("name", uc.RANDOM)
def test_random_lists_equal_the_reference_and_the_stream_continues(name):
    from elliot_b200.recommender import Random
    g = uc.case(name)
    data = uc.data_of(g)
    k = int(g["k"])
    m = _model(Random, data, seed=int(g["seed"]))
    for call in range(2):
        assert uc.same_dict(m.get_single_recommendation(None, k), uc.golden_dict(g, call)), call
        assert m._lists.stream.consumed == int(g[f"consumed_{call}"]), call


def test_random_stream_across_buffer_refills_and_users_subsets():
    """A buffer of 100 words forces refills in the middle of users; the result equals the oracle's for every call."""
    g = uc.case("random_42")
    data = uc.data_of(g)
    indptr, indices = uc.train_csr(data)
    lists = RandomLists(data, 42, DEV)
    lists.stream = ops.RandomStream(42, DEV, capacity=100)
    stream = oun.Stream(42)
    users = np.array([5, 2, 13, 17, 0, 5], np.int32)
    for call in range(3):
        want = oun.complement_select(oun.random_draws(stream, indptr, data.num_items, 10), indptr, indices,
                                     data.num_items)
        r = lists.stream.draws(10, lists.indptr, data.num_items)
        idx = ops.complement_select(r, lists.indptr, lists.train)
        assert np.array_equal(idx.cpu().numpy(), want), call
        sub = ops.complement_select(r, lists.indptr, lists.train, users=to_dev(users))
        assert np.array_equal(sub.cpu().numpy(), want[users]), call
        assert lists.stream.consumed == stream.consumed, call


@pytest.mark.parametrize("name", uc.CASES)
def test_device_metrics_equal_reference_on_lists_with_duplicates(name):
    g = uc.case(name)
    data = uc.data_of(g)
    names = g["metrics"].tolist()
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    for call in range(2 if "keys_1" in g else 1):
        recs = uc.golden_dict(g, call)
        if name == "mostpop":                                         # absent users: only the dict path can say so
            users = [u for u in recs if u in data.public_users]
        else:
            users = data.users
        idx = np.full((len(users), 10), -1, np.int32)
        for r, u in enumerate(users):
            row = [data.public_items[i] for i, _ in recs[u]]
            idx[r, :len(row)] = row
        priv = np.array([data.public_users[u] for u in users], np.int32)
        res = ev.eval_tensors(to_dev(idx), users=to_dev(priv))
        for c, k in enumerate(uc.CUTOFFS):
            for m, w in zip(names, g[f"values_{call}"][c].tolist()):
                got = res[k]["test_results"][m]
                assert abs(got - w) <= 1e-12 * max(1.0, abs(w)), (name, call, k, m, got, w)


# ---------------------------------------------------------------- run_experiment at C1 scale
c1 = c1h.c1_fixture("unpersonalized_c1.npz")


def _yaml(g, tsv, out, ev, key="MostPop"):
    extra = f"  external_models_path: {os.path.join(os.path.dirname(synth_c1.__file__), 'plugin.py')}\n"
    return synth_c1.unpersonalized_yaml(tsv, str(out), g["metrics"].tolist(), g["cutoffs"].tolist(), mostpop_key=key,
                                        extra=extra if key.startswith("external.") else "",
                                        model_extra=f"      b200_eval: {ev}\n")


@pytest.mark.parametrize("ev,key", [("host", "MostPop"), ("device", "MostPop"), ("host", "external.MostPop")])
def test_run_experiment_matches_the_reference_run(c1, ev, key):
    from elliot_b200 import run_experiment
    g, d, tsv = c1
    out = d / f"{key}_{ev}"
    os.makedirs(out, exist_ok=True)
    text = _yaml(g, tsv, out, ev, key)
    if ev == "device":
        text = text.replace("save_recs: True", "save_recs: False")
    (out / "cfg.yml").write_text(text)
    results = run_experiment(str(out / "cfg.yml"))
    assert [r["name"] for r in results] == ["MostPop", "Random_seed=42"]
    names = g["metrics"].tolist()
    for j, res in enumerate(results):
        for c, k in enumerate(g["cutoffs"].tolist()):
            for m, w in zip(names, g["test_metrics"][j, c].tolist()):
                got = res["test_results"][k][m]
                assert abs(got - w) <= 1e-12 * max(1.0, abs(w)), (key, ev, j, k, m, got, w)
    if ev == "device":
        c1h.assert_no_rec_files(out)
        return
    files = sorted(os.listdir(out / "recs"))
    assert files == g["rec_files"].tolist(), files
    for j, f in enumerate(files):
        lines = (out / "recs" / f).read_text().splitlines()
        assert len(lines) == int(g[f"n_lines_{j}"]), f
        want = g[f"lines_{j}"].tolist()
        assert lines[:len(want)] == want, f


@pytest.mark.parametrize("key", ["MostPop", "Random"])
def test_auc_is_refused_naming_the_model(c1, key):
    from elliot_b200 import run_experiment
    g, d, tsv = c1
    out = d / f"{key}_auc"
    os.makedirs(out, exist_ok=True)
    block = "      random_seed: 42\n" if key == "Random" else ""
    (out / "cfg.yml").write_text(synth_c1.experiment_yaml(tsv, str(out), key, block, metrics=("nDCG", "AUC")))
    with pytest.raises(Exception, match=f"{key} cannot evaluate AUC"):
        run_experiment(str(out / "cfg.yml"))
