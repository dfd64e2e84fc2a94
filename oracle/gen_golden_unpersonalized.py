#!/usr/bin/env python
"""Mint the MostPop and Random goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/unpersonalized_cases.npz
      the reference's own MostPop and Random classes (recommender/unpersonalized/), imported by file path through
      oracle/ref_stubs.py, on small train / test frames loaded by the reference's DataSet, with public ids that differ
      from the private ones.  Per case and call: the dict get_single_recommendation returned (its keys in order, each
      list's length, the public items and the scores, which must be Python ints), and the reference Evaluator's test
      metrics on that dict at every cutoff.  Cases:
        mostpop   popularity ties, items nobody rated, two users with |train_u| + k >= n_items whose PRIVATE ids are
                  the public ids of a later user (which keeps its list) and of an earlier one (which ends up with []),
                  and a user one short of the limit;
        random_*  seeds 42, 7 and 2024, each called twice (the stream continues); users with n_u = 0, 1, 3 < k, a
                  power of two (no rejection) and one more (the most rejection).
      Before saving, each dict is checked against oracle/unpersonalized.py.
  tests/golden/unpersonalized_c1.npz
      elliot.run.run_experiment on synth_c1.unpersonalized_yaml over the C1 synthetic file (MostPop and Random_seed=42,
      the evaluator's 23 list metrics at cutoffs 5 and 10): the test metrics of both models, each rec file's name and
      its lines for the first 400 users in file order, the dataset checksum and the run's wall time.

    python oracle/gen_golden_unpersonalized.py [--skip-c1] [--skip-cases]
"""
import argparse
import glob
import logging
import os
import shutil
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs, unpersonalized as oun  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402
from elliot_b200.evaluation import METRICS as EXTENDED  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
BASIC = ["nDCG", "HR", "Precision", "Recall"]
ALL = BASIC + list(EXTENDED)
K, CUTOFFS = 10, [5, 10]
RANDOM_SEEDS = (42, 7, 2024)


def _config(metrics):
    return SimpleNamespace(config_test=True, align_side_with_train=False, top_k=K,
                           evaluation=SimpleNamespace(simple_metrics=metrics, relevance_threshold=0,
                                                      paired_ttest=False, cutoffs=CUTOFFS))


def _frame(rows):
    rows = np.asarray(rows, np.int64).reshape(-1, 3)
    return pd.DataFrame({"userId": rows[:, 0], "itemId": rows[:, 1], "rating": rows[:, 2].astype(np.float64)})


def frames(seed, n_items, sizes, public):
    """Train rows in private-user order (the reference's DataSet numbers users by first appearance), items drawn with a
    skewed popularity (so that small counts tie) and every item rated by someone; test rows: up to 6 items outside
    each user's train row plus, now and then, a test-only item."""
    g = np.random.default_rng(seed)
    item_pub = 3000 + 7 * g.permutation(n_items)
    p = 1.0 / np.arange(1, n_items + 1) ** 0.7
    p /= p.sum()
    train, test = [], []
    rows = []
    for u, s in enumerate(sizes):
        its = g.choice(n_items, size=s, replace=False, p=p) if s < n_items else np.arange(n_items)
        rows.append(set(its.tolist()))
        train += [(public[u], item_pub[i], int(g.integers(1, 6))) for i in its]
    missing = set(range(n_items)) - set().union(*rows)
    for i in missing:                                   # every item is a train item of the user with the largest row
        u = int(np.argmax([s if s < n_items else -1 for s in sizes]))
        train.append((public[u], item_pub[i], 3))
        rows[u].add(i)
    for u in range(len(sizes)):
        free = sorted(set(range(n_items)) - rows[u])
        te = g.choice(free, size=min(6, len(free)), replace=False) if free else []
        test += [(public[u], item_pub[i], int(g.integers(1, 6))) for i in te]
        if u % 4 == 1 and len(free) > 6:               # (LAUC divides by the items outside train and test)
            test.append((public[u], 9999, 4))
    return _frame(train), _frame(test)


def dataset(tr, te, metrics):
    import elliot.dataset.dataset as ds
    return ds.DataSet(_config(metrics), (tr, te), SimpleNamespace())


def ref_model(cls, data, **params):
    """An instance of the reference class with its constructor body run (init_charger's framework part skipped)."""
    m = object.__new__(cls)
    m._data, m._params, m.logger = data, SimpleNamespace(**params), logging.getLogger("golden")
    m._num_items, m._num_users = data.num_items, data.num_users
    cls.__init__.__wrapped__(m, data, None, m._params)
    return m


def evaluate(data, recs, metrics):
    from elliot.evaluation.evaluator import Evaluator
    res = Evaluator(data, SimpleNamespace(meta=SimpleNamespace())).eval((recs, recs))
    return np.array([[float(res[k]["test_results"][m]) for m in metrics] for k in CUTOFFS])


def flat(recs):
    """keys, lengths, items, scores of a {key: [(item, score)]} dict, in its order; every score must be an int."""
    assert all(type(s) is int for lst in recs.values() for _, s in lst)
    return (np.array(list(recs), np.int64), np.array([len(v) for v in recs.values()], np.int64),
            np.array([i for v in recs.values() for i, _ in v], np.int64),
            np.array([s for v in recs.values() for _, s in v], np.int64))


def train_csr(data):
    m = data.sp_i_train.tocsr()
    m.sort_indices()
    return m.indptr.astype(np.int64), m.indices.astype(np.int64)


def expected_mostpop(data, rows, pop, skipped):
    r = {}
    for u in range(data.num_users):
        if skipped[u]:
            r[u] = []
        else:
            r[data.private_users[u]] = [(data.private_items[i], int(pop[u, j])) for j, i in enumerate(rows[u]) if i >= 0]
    return r


def case_mostpop(mod):
    n_items, n_users = 60, 40
    sizes = [int(x) for x in np.random.default_rng(5).integers(3, 25, n_users)]
    sizes[5], sizes[20], sizes[11] = 52, 50, 49            # |train_u| + k >= 60 for private 5 and 20; 11 is one short
    public = [500 + 7 * u for u in range(n_users)]
    public[30], public[3] = 5, 20                          # key 5 is written again later, key 20 was written earlier
    tr, te = frames(1, n_items, sizes, public)
    metrics = [m for m in ALL if m not in ("ARP", "APLT")]  # the reference divides by the length of user 3's [] there
    data = dataset(tr, te, metrics)
    assert data.users == public
    recs = ref_model(mod.MostPop, data).get_single_recommendation(data.allunrated_mask, K)
    indptr, indices = train_csr(data)
    rows, pop, skipped = oun.mostpop(indptr, indices, data.num_items, K)
    assert recs == expected_mostpop(data, rows, pop, skipped)
    assert recs[5] != [] and recs[20] == [] and 520 not in recs and 640 not in recs
    keys, lens, items, scores = flat(recs)
    return {"train": tr.values, "test": te.values, "metrics": np.array(metrics), "k": K, "seed": -1,
            "users": np.array(data.users, np.int64), "items": np.array(data.items, np.int64),
            "keys_0": keys, "lens_0": lens, "items_0": items, "scores_0": scores,
            "values_0": evaluate(data, recs, metrics)}


def case_random(mod, seed):
    n_items = 40
    sizes = [int(x) for x in np.random.default_rng(seed).integers(2, 30, 36)]
    sizes[2], sizes[5], sizes[9], sizes[13], sizes[17] = 40, 39, 37, 8, 7   # n_u = 0, 1, 3, 32, 33
    g = np.random.default_rng(seed + 1)
    public = (100 + 3 * g.permutation(len(sizes))).tolist()
    tr, te = frames(seed, n_items, sizes, public)
    metrics = [m for m in ALL if m not in ("ARP", "APLT")]  # the n_u = 0 user has test rows and an empty list
    data = dataset(tr, te, metrics)
    m = ref_model(mod.Random, data, random_seed=seed)
    assert m.name == f"Random_seed={seed}"
    indptr, indices = train_csr(data)
    stream = oun.Stream(seed)
    out = {"train": tr.values, "test": te.values, "metrics": np.array(metrics), "k": K, "seed": seed,
           "users": np.array(data.users, np.int64), "items": np.array(data.items, np.int64)}
    for call in range(2):
        recs = m.get_single_recommendation(data.allunrated_mask, K)
        idx = oun.complement_select(oun.random_draws(stream, indptr, data.num_items, K), indptr, indices, data.num_items)
        assert recs == {data.private_users[u]: [(data.private_items[i], 1) for i in idx[u] if i >= 0]
                        for u in range(data.num_users)}, (seed, call)
        keys, lens, items, scores = flat(recs)
        out.update({f"keys_{call}": keys, f"lens_{call}": lens, f"items_{call}": items, f"scores_{call}": scores,
                    f"values_{call}": evaluate(data, recs, metrics), f"consumed_{call}": stream.consumed})
    return out


def cases():
    base = os.path.join(ref_stubs.REF, "elliot", "recommender", "unpersonalized")
    mp = ref_stubs.load(os.path.join(base, "most_popular", "most_popular.py"), "ref_most_popular")
    rd = ref_stubs.load(os.path.join(base, "random_recommender", "Random.py"), "ref_random")
    mod = SimpleNamespace(MostPop=mp.MostPop, Random=rd.Random)
    out = {"mostpop": case_mostpop(mod)}
    for s in RANDOM_SEEDS:
        out[f"random_{s}"] = case_random(mod, s)
    flat_out = {f"{c}_{k}": v for c, d in out.items() for k, v in d.items()}
    np.savez_compressed(os.path.join(GOLD, "unpersonalized_cases.npz"), cases=np.array(list(out)), **flat_out)
    for c, d in out.items():
        dup = sum(len(set(d["items_0"][a:b])) < b - a for a, b in zip(np.cumsum(d["lens_0"]) - d["lens_0"], np.cumsum(d["lens_0"])))
        print(c, "users", len(d["keys_0"]), "lists with a duplicate", dup, flush=True)


def first_lines(path, keep=400):
    """The lines of the first `keep` users of a rec file, in file order."""
    with open(path) as fh:
        lines = fh.read().splitlines()
    users = list(dict.fromkeys(ln.split("\t")[0] for ln in lines))[:keep]
    sel = set(users)
    return np.array([ln for ln in lines if ln.split("\t")[0] in sel]), len(lines)


def c1_run():
    from elliot.evaluation.evaluator import Evaluator
    from elliot.run import run_experiment
    ref_stubs.install()
    tmp = tempfile.mkdtemp(prefix="c1_unpersonalized_")
    try:
        tsv = os.path.join(tmp, "dataset.tsv")
        checksum = synth_c1.write_tsv(tsv)
        logcfg = ref_stubs.write_logger_config(os.path.join(tmp, "logger_config.yml"))
        cfg = os.path.join(tmp, "cfg.yml")
        with open(cfg, "w") as fh:
            fh.write(synth_c1.unpersonalized_yaml(tsv, tmp, ALL, CUTOFFS, extra=f"  path_logger_config: {logcfg}\n"))
        evals, orig = [], Evaluator.eval

        def recording_eval(self, recommendations):        # pass-through: records what the reference computed
            res = orig(self, recommendations)
            evals.append([[float(res[k]["test_results"][m]) for m in ALL] for k in CUTOFFS])
            return res
        Evaluator.eval = recording_eval
        try:
            t0 = time.time()
            run_experiment(cfg)
            dt = time.time() - t0
        finally:
            Evaluator.eval = orig
        out = {"metrics": np.array(ALL), "cutoffs": np.array(CUTOFFS), "checksum": np.uint64(checksum),
               "reference_seconds": dt, "test_metrics": np.array(evals)}
        files = sorted(glob.glob(os.path.join(tmp, "recs", "*.tsv")))
        out["rec_files"] = np.array([os.path.basename(f) for f in files])
        for j, f in enumerate(files):
            out[f"lines_{j}"], out[f"n_lines_{j}"] = first_lines(f)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert len(evals) == 2 and list(out["rec_files"]) == ["MostPop.tsv", "Random_seed=42.tsv"], out["rec_files"]
    np.savez_compressed(os.path.join(GOLD, "unpersonalized_c1.npz"), **out)
    print(f"c1: {out['rec_files']}, run {dt:.1f} s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    ap.add_argument("--skip-cases", action="store_true")
    args = ap.parse_args()
    ref_stubs.install()
    logging.disable(logging.CRITICAL)
    if not args.skip_cases:
        cases()
    if not args.skip_c1:
        c1_run()


if __name__ == "__main__":
    main()
