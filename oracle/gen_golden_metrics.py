"""Golden values of the 19 list metrics the evaluator computes besides nDCG / HR / Precision / Recall, from the
UNMODIFIED reference Evaluator (elliot/evaluation/evaluator.py) run through oracle/ref_stubs.py.

tests/golden/metrics_cases.npz: three small datasets (train / validation / test frames) with test-only items, users with
test rows but no relevant item, users without test rows, short lists, relevance thresholds 0 and 3; the third case has
one empty list and asks for every metric but ARP and APLT (the reference divides by the list length there).  For each
case: the top-k lists as private-id arrays (-1 after the end of a list), every metric at cutoffs {1, 5, 10, top_k} for
validation and test, and every per-user metric's eval_user_metric() aligned to private users (NaN where absent).

tests/golden/metrics_c1.npz: the C1 synthetic file (elliot_b200/synth_c1.py, checksum recorded), split by the
reference's Splitter (random_subsampling 0.2, seed 42) and loaded by its DataSet; seeded popularity-skewed top-20 lists
without train items; every metric at {5, 10, 20}; the reference Evaluator's wall time for them on one host core.

    python oracle/gen_golden_metrics.py
"""
import logging
import os
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
ALL = ["nDCGRendle2020", "MRR", "MAP", "MAR", "F1", "LAUC", "NumRetrieved", "EPC", "EFD", "ARP", "APLT", "ACLT",
       "PopREO", "PopRSP", "ItemCoverage", "UserCoverage", "UserCoverageAtN", "Gini", "SEntropy"]
PER_USER = ["nDCGRendle2020", "MRR", "MAP", "MAR", "F1", "LAUC", "NumRetrieved", "EPC", "EFD", "ARP", "APLT", "ACLT"]


def _config(top_k, cutoffs, thr, metrics):
    return SimpleNamespace(config_test=True, align_side_with_train=False, top_k=top_k,
                           evaluation=SimpleNamespace(simple_metrics=metrics, relevance_threshold=thr,
                                                      paired_ttest=False, cutoffs=cutoffs))


def _frame(rows):
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": rows[:, 0].astype(np.int64), "itemId": rows[:, 1].astype(np.int64), "rating": rows[:, 2]})


def _lists(g, data, top_k, short_every=0, empty_user=None):
    """Popularity-skewed lists of distinct train items the user has not rated, as {public user: [(item, score)]}."""
    n_items = data.num_items
    pop = np.asarray(data.sp_i_train.sum(axis=0)).ravel() + 1.0
    p = pop / pop.sum()
    recs = {}
    for pu, u in enumerate(data.users):
        seen = set(data.i_train_dict[pu])
        cand = [i for i in g.choice(n_items, size=min(n_items, 4 * top_k), replace=False, p=p) if i not in seen]
        n = top_k
        if short_every and pu % short_every == 3:
            n = int(g.integers(1, top_k))
        if u == empty_user:
            n = 0
        recs[u] = [(data.private_items[i], float(top_k - q)) for q, i in enumerate(cand[:n])]
    return recs


def _as_array(data, recs, top_k):
    a = np.full((data.num_users, top_k), -1, np.int32)
    for u, lst in recs.items():
        row = [data.public_items[i] for i, _ in lst]
        a[data.public_users[u], :len(row)] = row
    return a


def _evaluate(data, recs, metrics):
    """The reference Evaluator's results for every cutoff, and each per-user metric's eval_user_metric() on the same
    user filter and evaluation objects the Evaluator uses (evaluator.py:117-122)."""
    from elliot.evaluation import metrics as M
    from elliot.evaluation.evaluator import Evaluator
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    res = ev.eval((recs, recs))
    cut = data.config.evaluation.cutoffs
    vals = np.array([[[float(res[k][s][m]) for m in metrics] for s in ("val_results", "test_results")] for k in cut])
    per = np.full((len(cut), 2, len(PER_USER), data.num_users), np.nan)
    for c, k in enumerate(cut):
        for s, (test_data, eval_objs) in enumerate(ev._get_test_data()):
            eval_objs.cutoff = k
            kept = {u: r for u, r in recs.items() if test_data.get(u, [])}
            for j, name in enumerate(PER_USER):
                if name not in metrics:
                    continue
                for u, v in M.parse_metric(name)(kept, data.config, ev._params, eval_objs).eval_user_metric().items():
                    per[c, s, j, data.public_users[u]] = v
    return vals, per


def make_case(seed, n_users, n_items, thr, top_k, metrics, empty):
    import elliot.dataset.dataset as ds
    g = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.9
    pop /= pop.sum()
    tr, va, te = [], [], []
    for u in range(n_users):
        uid = 7 + 3 * u
        its = g.choice(n_items + 15, size=int(g.integers(6, 30)), replace=False,
                       p=np.r_[pop * 0.9, np.full(15, 0.1 / 15)])          # ids >= n_items: rare, mostly test-only
        its = 1000 + 5 * its
        rat = g.integers(1, 6, size=its.size).astype(np.float64)
        if u % 11 == 5:
            rat[:] = np.minimum(rat, 2.0)                                   # test rows, none relevant at threshold 3
        n_tr = max(3, int(0.6 * its.size))
        n_va = (its.size - n_tr) // 2
        tr += [(uid, i, r) for i, r in zip(its[:n_tr], rat[:n_tr])]
        if u % 13 != 2:                                                     # some users have no validation rows
            va += [(uid, i, r) for i, r in zip(its[n_tr:n_tr + n_va], rat[n_tr:n_tr + n_va])]
        if u % 17 != 4:                                                     # ... or no test rows
            te += [(uid, i, r) for i, r in zip(its[n_tr + n_va:], rat[n_tr + n_va:])]
    tr, va, te = (np.array(x) for x in (tr, va, te))
    g.shuffle(tr); g.shuffle(va); g.shuffle(te)
    cutoffs = sorted({1, 5, 10, top_k})
    data = ds.DataSet(_config(top_k, cutoffs, thr, metrics), (_frame(tr), _frame(va), _frame(te)), SimpleNamespace())
    empty_user = data.users[[pu for pu in range(data.num_users) if data.test_dict[data.users[pu]]][0]] if empty else None
    recs = _lists(g, data, top_k, short_every=7, empty_user=empty_user)
    vals, per = _evaluate(data, recs, metrics)
    from elliot.evaluation.popularity_utils import Popularity
    short_head = np.array([data.public_items[i] for i in Popularity(data).get_short_head()], np.int64)
    return dict(short_head=short_head, train=tr, val=va, test=te, thr=thr, top_k=top_k, cutoffs=np.array(cutoffs), metrics=np.array(metrics),
                users=np.array(data.users, np.int64), items=np.array(data.items, np.int64),
                rec_idx=_as_array(data, recs, top_k), values=vals, per_user=per)


def make_cases():
    no_div = [m for m in ALL if m not in ("ARP", "APLT")]
    cases = {"a": make_case(11, 220, 160, 0, 20, ALL, False),
             "b": make_case(12, 260, 200, 3, 15, ALL, False),
             "c": make_case(13, 180, 120, 3, 10, no_div, True)}
    out = {f"{c}_{k}": v for c, d in cases.items() for k, v in d.items()}
    np.savez_compressed(os.path.join(OUT, "metrics_cases.npz"), cases=np.array(sorted(cases)), **out)
    for c, d in cases.items():
        print(c, dict(zip(d["metrics"].tolist(), np.round(d["values"][-1, 1], 6).tolist())))


def make_c1():
    import elliot.dataset.dataset as ds
    from elliot.splitter.base_splitter import Splitter
    from elliot_b200 import synth_c1
    from elliot.evaluation.evaluator import Evaluator
    with tempfile.TemporaryDirectory() as tmp:
        tsv = os.path.join(tmp, "dataset.tsv")
        checksum = synth_c1.write_tsv(tsv)
        df = pd.read_csv(tsv, sep="\t", header=None, names=["userId", "itemId", "rating", "timestamp"])
    ns = SimpleNamespace(test_splitting=SimpleNamespace(strategy="random_subsampling", test_ratio=0.2))
    (train, test), = Splitter(df, ns, 42).process_splitting()
    top_k, cutoffs = 20, [5, 10, 20]
    data = ds.DataSet(_config(top_k, cutoffs, 0, ALL), (train, test), SimpleNamespace())
    g = np.random.default_rng(2024)
    recs = _lists(g, data, top_k)
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    t0 = time.perf_counter()
    res = ev.eval((recs, recs))
    dt = time.perf_counter() - t0
    vals = np.array([[float(res[k]["test_results"][m]) for m in ALL] for k in cutoffs])
    np.savez_compressed(os.path.join(OUT, "metrics_c1.npz"), checksum=checksum, top_k=top_k, cutoffs=np.array(cutoffs),
                        metrics=np.array(ALL), users=np.array(data.users, np.int64), items=np.array(data.items, np.int64),
                        rec_idx=_as_array(data, recs, top_k), values=vals, reference_seconds=dt)
    print("c1", data.num_users, data.num_items, f"{dt:.1f} s", dict(zip(ALL, np.round(vals[-1], 6).tolist())))


if __name__ == "__main__":
    ref_stubs.install()
    logging.disable(logging.CRITICAL)
    make_cases()
    make_c1()
