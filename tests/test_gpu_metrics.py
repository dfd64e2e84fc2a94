"""eb_eval_metrics_f64 / Evaluator.eval_tensors for the 19 list metrics beyond nDCG / HR / Precision / Recall: the device
against the reference Evaluator's goldens (tests/golden/metrics_*.npz) and per-user values, against the host mirror on
random lists, bit-identical reruns, empty and all-skipped inputs, and one run_experiment at C1 with both evaluation
paths."""
import numpy as np
import pandas as pd
import pytest
import torch

import c1_harness as c1h
from c1_harness import DEV
from elliot_b200 import ops
from elliot_b200.dataset import DataSet
from elliot_b200.evaluation import METRICS, N_SLOTS, PER_USER, S_EMPTY, S_GINI_S, S_ITEMCOV, S_UCOV, S_UCOV_N, Evaluator, \
    host_metric_sums
from test_metrics_host import CASES, GOLD, INTEGER, assert_close, case_data, config

pytestmark = pytest.mark.gpu
EXACT = [S_UCOV, S_UCOV_N, S_EMPTY, S_ITEMCOV, S_GINI_S, 0, 10, 11, 12, 13, 14, 17, 18, 19, 20, 21, 24]   # integer slots


def _slots(ev, which, k, idx, users=None, per_user=False):
    s, per = ops.eval_topk_metrics(torch.from_numpy(np.ascontiguousarray(idx)).to(DEV), k,
                                   *ev._metric_device_set(which, k, torch.device(DEV)),
                                   users=None if users is None else torch.from_numpy(users).to(DEV), per_user=per_user)
    return s.cpu().numpy(), None if per is None else per.cpu().numpy()


def _assert_slots(got, want, what):
    assert np.array_equal(got[EXACT], want[EXACT]), (what, got[EXACT], want[EXACT])
    rest = np.setdiff1d(np.arange(N_SLOTS), EXACT)
    np.testing.assert_allclose(got[rest], want[rest], rtol=1e-12, atol=1e-300, err_msg=str(what))


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_equals_reference_evaluator(case):
    g, data, ev = case_data(case)
    names = g["metrics"].tolist()
    res = ev.eval_tensors(torch.from_numpy(g["rec_idx"]).to(DEV))
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, split in enumerate(("val_results", "test_results")):
            assert list(res[k][split]) == names
            assert_close(res[k][split], dict(zip(names, g["values"][c, s].tolist())), (case, k, split))


def test_device_equals_reference_at_c1():
    import os
    import tempfile
    from elliot_b200 import synth_c1
    from elliot_b200.run import _read, split_random_subsampling
    g = np.load(os.path.join(GOLD, "metrics_c1.npz"))
    with tempfile.TemporaryDirectory() as tmp:
        tsv = os.path.join(tmp, "dataset.tsv")
        assert synth_c1.write_tsv(tsv) == int(g["checksum"])
        df = _read(tsv, False)
    (train, test), = split_random_subsampling(df, 0.2, 42)
    names = g["metrics"].tolist()
    data = DataSet(config(int(g["top_k"]), g["cutoffs"].tolist(), 0, names), (train, test))
    ev = Evaluator(data, None)
    res = ev.eval_tensors(torch.from_numpy(g["rec_idx"]).to(DEV))
    for c, k in enumerate(g["cutoffs"].tolist()):
        assert_close(res[k]["test_results"], dict(zip(names, g["values"][c].tolist())), ("c1", k))


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_per_user_values_equal_reference(case):
    g, data, ev = case_data(case)
    asked = [j for j, m in enumerate(PER_USER) if m in g["metrics"].tolist()]
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, which in enumerate(("val", "test")):
            _, per = _slots(ev, which, k, g["rec_idx"], per_user=True)
            want = g["per_user"][c, s].T
            np.testing.assert_array_equal(np.isnan(per[:, asked]), np.isnan(want[:, asked]))
            np.testing.assert_allclose(per[:, asked], want[:, asked], rtol=1e-12, atol=1e-15)


def _random_case(k, seed):
    rs = np.random.RandomState(seed)
    n_users, n_items = 400, max(300, k + 200)
    tr = [(u, i, 1.0) for u in range(n_users) for i in rs.choice(n_items, rs.randint(1, 8), replace=False)]
    tr += [(i % n_users, i, 1.0) for i in range(n_items)]             # every item is a train item: lists up to k fit
    te = []
    for u in range(n_users):
        m = 0 if u % 7 == 0 else rs.randint(1, 40)                   # some users have no test rows at all
        for i in rs.choice(n_items + 20, m, replace=False):          # ids >= n_items never occur in training
            te.append((u, i, float(rs.randint(1, 6))))
    f = lambda a: pd.DataFrame({"userId": [x[0] for x in a], "itemId": [x[1] for x in a], "rating": [x[2] for x in a]})
    data = DataSet(config(k, [k], 3, METRICS), (f(tr), f(te)))
    idx = np.stack([rs.permutation(data.num_items)[:k] for _ in range(data.num_users)]).astype(np.int32)
    ends = np.where(rs.rand(data.num_users) < 0.2, rs.randint(0, k + 1, data.num_users), k)   # short and empty lists
    idx[np.arange(k)[None, :] >= ends[:, None]] = -1
    return rs, data, Evaluator(data, None), idx


@pytest.mark.parametrize("k", [1, 5, 10, 16, 50, 100, 1024])
def test_device_equals_host_mirror_on_random_lists(k):
    rs, data, ev, idx = _random_case(k, k)
    tab, cs = ev._tables("test"), ev._sets["test"]
    want, want_pu = host_metric_sums(tab, cs, np.arange(data.num_users), idx, k, per_user=True)
    got, got_pu = _slots(ev, "test", k, idx, per_user=True)
    _assert_slots(got, want, k)
    np.testing.assert_array_equal(np.isnan(got_pu), np.isnan(want_pu))
    np.testing.assert_allclose(got_pu, want_pu, rtol=1e-12, atol=1e-15)
    # explicit user ids: a shuffled subset of rows
    sel = rs.permutation(data.num_users)[:150].astype(np.int32)
    sub, _ = _slots(ev, "test", k, idx[sel], users=sel)
    _assert_slots(sub, host_metric_sums(tab, cs, sel.astype(np.int64), idx[sel], k)[0], (k, "users"))
    # deterministic: the same bits on a second launch
    again, _ = _slots(ev, "test", k, idx[sel], users=sel)
    assert np.array_equal(again, sub)


def test_empty_input_and_all_skipped():
    rs, data, ev, idx = _random_case(10, 3)
    s, _ = _slots(ev, "test", 10, idx[:0])
    assert s.tolist() == [0.0] * N_SLOTS
    no_rows = np.flatnonzero(ev._tables("test").user_info[:, 0] == 0).astype(np.int32)
    assert no_rows.size
    s, per = _slots(ev, "test", 10, idx[no_rows], users=no_rows, per_user=True)
    assert s.tolist() == [0.0] * N_SLOTS and bool(np.isnan(per).all())
    assert all(v == 0 for v in ev_values(ev, idx[no_rows], no_rows).values())


def ev_values(ev, idx, users):
    return ev.eval_tensors(torch.from_numpy(idx).to(DEV), users=torch.from_numpy(users).to(DEV))[10]["test_results"]


# ---------------------------------------------------------------- run_experiment at C1 scale
c1 = c1h.c1_fixture("ease_c1.npz")
ALL = ["nDCG", "nDCGRendle2020", "HR", "Precision", "Recall", "LAUC", "F1", "MAP", "MAR", "MRR", "NumRetrieved", "ACLT",
       "APLT", "ARP", "PopREO", "PopRSP", "ItemCoverage", "UserCoverage", "UserCoverageAtN", "Gini", "SEntropy", "EFD",
       "EPC"]


def test_run_experiment_with_every_metric_on_both_paths(c1):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    res = {}
    for ev in ("host", "device"):
        out = d / f"all_{ev}"
        text = synth_c1.ease_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n")
        text = text.replace("simple_metrics: [nDCG, HR, Precision, Recall]", f"simple_metrics: [{', '.join(ALL)}]")
        res[ev] = c1h.run(out, text, ev == "device")
        c1h.assert_metrics(res[ev], g["metrics"].tolist(), g["test_metrics"], ev)
    host, dev = res["host"]["test_results"][10], res["device"]["test_results"][10]
    assert list(host) == ALL and list(dev) == ALL
    for m in ALL:
        if m in INTEGER:
            assert host[m] == dev[m], m
        else:
            assert abs(host[m] - dev[m]) <= 1e-12 * max(1.0, abs(host[m])), (m, host[m], dev[m])
