"""Golden values of MAE, MSE and RMSE from the UNMODIFIED reference Evaluator (elliot/evaluation/evaluator.py,
metrics/rating/{mae,mse,rmse}) run through oracle/ref_stubs.py.

Every user's list is the reference's full list (get_top_k with k = num_items): the items outside its train profile by
(score desc, private item asc), then its train items with score -inf.  Scores are s = U V^T + b_i + b_u + g with small
integer tables and g = 0.5, exact in fp32 in any summation order.  Those lists go to the reference Evaluator at cutoffs
{5, 10}.

tests/golden/rating_metrics_cases.npz: the datasets of oracle/gen_golden_auc.py's cases (thresholds 0 and 3, test-only
items, users with test rows but no relevant item, users without test rows, a validation split); "inf" adds, at threshold
3, a relevant test row for an item of the user's train profile (its -inf score makes MAE / MSE / RMSE inf), and
"no_relevant" has no relevant test item at all (ZeroDivisionError, recorded as the case's `error`).

tests/golden/rating_metrics_c1.npz: the same on the C1 rows (elliot_b200/synth_c1.py) at threshold 3 with d = 2 integer
tables: a seeded 20 % test split whose test rows are kept for the first 300 users only (the reference's pure-Python
metrics walk every full list, 3 706 entries per user).  The rows are rebuilt by c1_frames(), not stored.

    python oracle/gen_golden_rating_metrics.py
"""
import logging
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import gen_golden_auc as auc_cases  # noqa: E402
from oracle import ref_stubs  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
NAMES = ["MAE", "MSE", "RMSE"]
CUTOFFS = [5, 10]
G_BIAS = 0.5


def _config(thr):
    return SimpleNamespace(config_test=True, align_side_with_train=False, top_k=10,
                           evaluation=SimpleNamespace(simple_metrics=NAMES, relevance_threshold=thr, paired_ttest=False,
                                                      cutoffs=CUTOFFS))


def full_lists(data, S):
    """Private-id full lists with their scores: non-train items by (score desc, item asc), then train items at -inf."""
    lists, scores = [], []
    for pu in range(data.num_users):
        seen = set(data.i_train_dict[pu])
        items = sorted((i for i in range(data.num_items) if i not in seen), key=lambda i: (-S[pu, i], i))
        tail = sorted(seen)
        lists.append(items + tail)
        scores.append([float(S[pu, i]) for i in items] + [-np.inf] * len(tail))
    return lists, scores


def _evaluate(data, lists, scores):
    from elliot.evaluation.evaluator import Evaluator
    recs = {data.users[pu]: [(data.items[i], v) for i, v in zip(lst, sc)] for pu, (lst, sc) in enumerate(zip(lists, scores))}
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    try:
        res = ev.eval((recs, recs))
    except ZeroDivisionError:
        return np.full((len(CUTOFFS), 2, len(NAMES)), np.nan), "ZeroDivisionError"
    return np.array([[[float(res[k][s][m]) for m in NAMES] for s in ("val_results", "test_results")]
                     for k in CUTOFFS]), ""


def tables(g, data, d):
    U = g.integers(-2, 3, size=(data.num_users, d)).astype(np.float64)
    V = g.integers(-2, 3, size=(data.num_items, d)).astype(np.float64)
    bi = g.integers(-1, 2, size=data.num_items).astype(np.float64)
    bu = g.integers(-1, 2, size=data.num_users).astype(np.float64)
    return U, V, bi, bu


def make_case(seed, n_users, n_items, thr, d=3, edit=None, overlap=False):
    import elliot.dataset.dataset as ds
    g = np.random.default_rng(seed)
    tr, va, te = auc_cases._interactions(g, n_users, n_items, -1)
    if edit is not None:
        tr, va, te = edit(tr, va, te)
    seen = set(map(tuple, tr[:, :2].tolist()))
    va, te = (np.array([r for r in a if (r[0], r[1]) not in seen]).reshape(-1, 3) for a in (va, te))
    if edit is None:                                    # relevant test-only items
        users = np.unique(tr[:, 0])
        te = np.r_[te, [(u, 900000 + 5 * j, 4.0) for j, u in enumerate(users) if j % 9 == 1]]
    if overlap:                                         # one relevant test row whose item is in the user's train profile
        u0 = te[0, 0]
        item = tr[tr[:, 0] == u0][0, 1]
        te = np.r_[te, [(u0, item, 5.0)]]
    g.shuffle(tr); g.shuffle(va); g.shuffle(te)
    data = ds.DataSet(_config(thr), (auc_cases._frame(tr), auc_cases._frame(va), auc_cases._frame(te)), SimpleNamespace())
    U, V, bi, bu = tables(g, data, d)
    S = U @ V.T + bi[None, :] + bu[:, None] + G_BIAS
    lists, scores = full_lists(data, S)
    vals, err = _evaluate(data, lists, scores)
    return dict(train=tr, val=va, test=te, thr=thr, U=U, V=V, bi=bi, bu=bu, g=G_BIAS, users=np.array(data.users, np.int64),
                items=np.array(data.items, np.int64), cutoffs=np.array(CUTOFFS), metrics=np.array(NAMES), values=vals,
                error=np.array(err))


def _no_relevant(tr, va, te):
    """Every test and validation rating below 3."""
    va, te = va.copy(), te.copy()
    va[:, 2] = np.minimum(va[:, 2], 2.0); te[:, 2] = np.minimum(te[:, 2], 2.0)
    return tr, va, te


def make_cases():
    cases = {"thr0": make_case(31, 120, 90, 0),
             "thr3": make_case(32, 150, 110, 3, d=4),
             "inf": make_case(33, 80, 70, 3, overlap=True),
             "no_relevant": make_case(34, 60, 50, 3, edit=_no_relevant)}
    out = {f"{c}_{k}": v for c, d in cases.items() for k, v in d.items()}
    np.savez_compressed(os.path.join(OUT, "rating_metrics_cases.npz"), cases=np.array(sorted(cases)), **out)
    for c, d in cases.items():
        print(c, d["error"] or d["values"][-1].tolist())


C1_SPLIT_SEED, C1_KEEP = 7, 300


def c1_frames():
    """(train rows, test rows) of the C1 golden: a seeded 20 % test split of synth_c1.rows(), test rows kept for the first
    C1_KEEP users only; and the generator, positioned for the tables."""
    from elliot_b200 import synth_c1
    u, i, r = synth_c1.rows()
    g = np.random.default_rng(C1_SPLIT_SEED)
    test = g.random(u.size) < 0.2
    tr = np.stack([u[~test], i[~test], r[~test]], 1).astype(np.float64)
    te = np.stack([u[test], i[test], r[test]], 1).astype(np.float64)
    return tr, te[np.isin(te[:, 0], np.unique(u)[:C1_KEEP])], g


def make_c1():
    """The frames are rebuilt from synth_c1 by c1_frames (its checksum is stored); the golden keeps the tables."""
    import elliot.dataset.dataset as ds
    from elliot_b200 import synth_c1
    tr, te, g = c1_frames()
    data = ds.DataSet(_config(3), (auc_cases._frame(tr), auc_cases._frame(te)), SimpleNamespace())
    U, V, bi, bu = tables(g, data, 2)
    S = U @ V.T + bi[None, :] + bu[:, None] + G_BIAS
    lists, scores = full_lists(data, S)
    vals, err = _evaluate(data, lists, scores)
    assert not err
    np.savez_compressed(os.path.join(OUT, "rating_metrics_c1.npz"), checksum=np.uint64(synth_c1.checksum(*synth_c1.rows())),
                        thr=3, U=U.astype(np.int8), V=V.astype(np.int8), bi=bi.astype(np.int8), bu=bu.astype(np.int8),
                        g=G_BIAS, users=np.array(data.users, np.int64), items=np.array(data.items, np.int64),
                        cutoffs=np.array(CUTOFFS), metrics=np.array(NAMES), values=vals)
    print("c1", vals[-1].tolist())


if __name__ == "__main__":
    ref_stubs.install()
    logging.disable(logging.CRITICAL)
    make_cases()
    make_c1()
