"""Golden values of AUC and GAUC from the UNMODIFIED reference Evaluator (elliot/evaluation/evaluator.py, auc.py,
gauc.py) run through oracle/ref_stubs.py.

tests/golden/auc_cases.npz: small datasets (train / validation / test frames) with small-integer factor tables, so every
score is an exact integer in any summation order and ties between items are common.  Each user's full list is every
item outside its train profile, ordered by (score desc, private item asc): the order ops.score_topk(k=n_items) lists
them in.  Those lists go to the reference Evaluator at cutoffs {5, 10}.  The cases cover ties, test-only items, users
with test rows but no relevant item, thresholds 0 and 3, a user with more relevant items than the rank kernel holds in
one shared-memory chunk, a validation split, no positive in any list (AUC = np.average([]) = NaN) and neg_u = 0
(ZeroDivisionError, recorded as the case's `error`).

tests/golden/auc_c1.npz: elliot.run.run_experiment on the C1 BPRMF block (synth_c1.yaml_text, factors 64) for one epoch
with AUC and GAUC added to the metrics and save_recs off: every metric of the one evaluation, and the wall time of the
reference Evaluator's eval() for it on one host core (a host timing).

    python oracle/gen_golden_auc.py [--cases-only]
"""
import argparse
import logging
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
NAMES = ["AUC", "GAUC"]
CUTOFFS = [5, 10]


def _config(thr):
    return SimpleNamespace(config_test=True, align_side_with_train=False, top_k=10,
                           evaluation=SimpleNamespace(simple_metrics=NAMES, relevance_threshold=thr, paired_ttest=False,
                                                      cutoffs=CUTOFFS))


def _frame(rows):
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": rows[:, 0].astype(np.int64), "itemId": rows[:, 1].astype(np.int64), "rating": rows[:, 2]})


def _interactions(g, n_users, n_items, big_user):
    """(train, val, test) rows: public ids 7 + 3u and 1000 + 5i, ids >= n_items rare and mostly test-only."""
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.9
    pop /= pop.sum()
    tr, va, te = [], [], []
    for u in range(n_users):
        uid = 7 + 3 * u
        size = int(0.8 * n_items) if u == big_user else int(g.integers(6, 30))
        p = np.full(n_items + 15, 1.0 / (n_items + 15)) if u == big_user else np.r_[pop * 0.9, np.full(15, 0.1 / 15)]
        its = 1000 + 5 * g.choice(n_items + 15, size=size, replace=False, p=p)
        rat = g.integers(1, 6, size=its.size).astype(np.float64)
        if u % 11 == 5:
            rat[:] = np.minimum(rat, 2.0)                                   # test rows, none relevant at threshold 3
        n_tr = max(3, int(0.6 * its.size))
        n_va = (its.size - n_tr) // 2
        if u == big_user:                                                   # most of its rows are test rows
            n_tr = n_va = int(0.1 * its.size)
        tr += [(uid, i, r) for i, r in zip(its[:n_tr], rat[:n_tr])]
        if u % 13 != 2:                                                     # some users have no validation rows
            va += [(uid, i, r) for i, r in zip(its[n_tr:n_tr + n_va], rat[n_tr:n_tr + n_va])]
        if u % 17 != 4:                                                     # ... or no test rows
            te += [(uid, i, r) for i, r in zip(its[n_tr + n_va:], rat[n_tr + n_va:])]
    for i in range(n_items):                                                # every item is a train item of someone
        tr.append((7 + 3 * (i % n_users), 1000 + 5 * i, 4.0))
    return _dedup(tr), np.array(va), np.array(te)


def _dedup(rows):
    seen, out = set(), []
    for r in rows:
        if (r[0], r[1]) not in seen:
            seen.add((r[0], r[1]))
            out.append(r)
    return np.array(out)


def full_lists(data, U, V, b):
    """Private-id full lists: items outside the train profile by (score desc, item asc); integer scores."""
    S = U @ V.T + b[None, :]
    out = []
    for pu in range(data.num_users):
        seen = set(data.i_train_dict[pu])
        items = [i for i in range(data.num_items) if i not in seen]
        out.append(sorted(items, key=lambda i: (-S[pu, i], i)))
    return out, S


def _evaluate(data, lists, S):
    """The reference Evaluator's AUC / GAUC for each cutoff and split, or the name of the exception it raises."""
    from elliot.evaluation.evaluator import Evaluator
    recs = {data.users[pu]: [(data.items[i], float(S[pu, i])) for i in lst] for pu, lst in enumerate(lists)}
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    try:
        res = ev.eval((recs, recs))
    except ZeroDivisionError:
        return np.full((len(CUTOFFS), 2, len(NAMES)), np.nan), "ZeroDivisionError"
    return np.array([[[float(res[k][s][m]) for m in NAMES] for s in ("val_results", "test_results")]
                     for k in CUTOFFS]), ""


def make_case(seed, n_users, n_items, thr, d=3, big_user=-1, edit=None):
    import elliot.dataset.dataset as ds
    g = np.random.default_rng(seed)
    tr, va, te = _interactions(g, n_users, n_items, big_user)
    if edit is not None:
        tr, va, te = edit(tr, va, te)
    seen = set(map(tuple, tr[:, :2].tolist()))                              # no (user, item) in train and in a split
    va, te = (np.array([r for r in a if (r[0], r[1]) not in seen]).reshape(-1, 3) for a in (va, te))
    g.shuffle(tr); g.shuffle(va); g.shuffle(te)
    data = ds.DataSet(_config(thr), (_frame(tr), _frame(va), _frame(te)), SimpleNamespace())
    U = g.integers(-2, 3, size=(data.num_users, d)).astype(np.float64)
    V = g.integers(-2, 3, size=(data.num_items, d)).astype(np.float64)
    b = g.integers(-1, 2, size=data.num_items).astype(np.float64)
    lists, S = full_lists(data, U, V, b)
    vals, err = _evaluate(data, lists, S)
    lens = np.array([len(x) for x in lists], np.int64)
    return dict(train=tr, val=va, test=te, thr=thr, U=U, V=V, bias=b, users=np.array(data.users, np.int64),
                items=np.array(data.items, np.int64), list_indptr=np.r_[0, np.cumsum(lens)],
                list_items=np.concatenate(lists).astype(np.int32), cutoffs=np.array(CUTOFFS), metrics=np.array(NAMES),
                values=vals, error=np.array(err))


def _no_positive(tr, va, te):
    """Every relevant row is a test-only item: lists hold no positive."""
    known = np.unique(tr[:, 1])
    new = known.max() + 5 * np.arange(1, 8)
    users = np.unique(tr[:, 0])
    extra = lambda off: np.array([(u, new[(j + off) % 7], 5.0) for j, u in enumerate(users) if j % 3 != 1])
    return tr, np.r_[va[~np.isin(va[:, 1], known)], extra(0)], np.r_[te[~np.isin(te[:, 1], known)], extra(3)]


def _zero_neg(tr, va, te):
    """User 7 trains on every item but two, which are in its test rows with a test-only item: neg = 0 with positives."""
    items = np.unique(tr[:, 1])
    tr = np.r_[tr[tr[:, 0] != 7], [(7, i, 4.0) for i in items[2:]]]
    te = np.r_[te[te[:, 0] != 7], [(7, items[0], 5.0), (7, items[1], 5.0), (7, items.max() + 5, 5.0)]]
    return tr, va[va[:, 0] != 7], te


def make_cases():
    cases = {"ties": make_case(21, 120, 90, 0),
             "thr3": make_case(22, 150, 110, 3, d=4),
             "big": make_case(23, 40, 2600, 0, d=2, big_user=5),
             "no_positive": make_case(24, 60, 50, 0, edit=_no_positive),
             "zero_neg": make_case(25, 50, 40, 0, edit=_zero_neg)}
    out = {f"{c}_{k}": v for c, d in cases.items() for k, v in d.items()}
    np.savez_compressed(os.path.join(OUT, "auc_cases.npz"), cases=np.array(sorted(cases)), **out)
    for c, d in cases.items():
        print(c, d["error"] or np.round(d["values"][-1], 6).tolist())


def make_c1():
    from elliot.evaluation.evaluator import Evaluator
    from elliot_b200 import synth_c1
    ref_stubs.install()
    metrics = ref_stubs.METRICS + NAMES
    evals, seconds = [], []
    orig_eval = Evaluator.eval

    def recording_eval(self, recommendations):             # pass-through: records every metric and the eval time
        t0 = time.perf_counter()
        res = orig_eval(self, recommendations)
        seconds.append(time.perf_counter() - t0)
        k = list(res.keys())[0]
        evals.append([float(res[k]["test_results"][m]) for m in metrics])
        return res
    Evaluator.eval = recording_eval
    try:
        _, recs, checksum, dt = ref_stubs.run_c1(lambda tsv, d, extra: synth_c1.yaml_text(
            tsv, d, "BPRMF", 1, 64, extra=extra, save_recs=False, metrics=metrics))
    finally:
        Evaluator.eval = orig_eval
    assert not recs and len(evals) == 1
    np.savez_compressed(os.path.join(OUT, "auc_c1.npz"), metrics=np.array(metrics), values=np.array(evals[0]), epochs=1,
                        factors=64, checksum=np.uint64(checksum), reference_eval_seconds=seconds[0],
                        reference_seconds=dt)
    print("c1", dict(zip(metrics, np.round(evals[0], 6).tolist())), f"eval {seconds[0]:.1f} s, run {dt:.0f} s")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases-only", action="store_true")
    args = ap.parse_args()
    ref_stubs.install()
    logging.disable(logging.CRITICAL)
    make_cases()
    if not args.cases_only:
        make_c1()
