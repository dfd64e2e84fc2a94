"""Golden values of the clustered fairness metrics (BiasDisparityBR / BS / BD, User/ItemMADrating, User/ItemMADranking,
REO, RSP) from the UNMODIFIED reference Evaluator (elliot/evaluation/evaluator.py, complex_metrics) run through
oracle/ref_stubs.py.

tests/golden/fairness_cases.npz: four small datasets in the shape of gen_golden_metrics.make_case (test-only items, users
without test rows, users with test rows but no relevant item at threshold 3, short lists, one empty list, lists with
repeated items, float scores).  Their clustering tables are stored in the npz: user files that miss dataset users and
list users the dataset lacks, item files that list test-only items and ids outside the catalogue, a user cluster that
ends up empty, a single-cluster item file, one case without any clustering file and one item clustering of 300
clusters.  Every entry's keys and values at cutoffs {1, 5, 10, top_k} for validation and test.

tests/golden/fairness_c1.npz: the C1 synthetic file (checksum recorded), split and loaded by the reference, with the
reference's own data/movielens_1m/u_happy.tsv and i_pop.tsv as data fixtures; seeded top-20 lists with float scores
(c1_lists: drawn from the dataset alone, so the tests redraw them; only their checksums are stored);
all nine metrics at {5, 10, 20} and the reference Evaluator's wall time for them on one host core.  Also the reference's
run_experiment on the same file with a MostPop block and the advanced configuration's complex entry (UserMADrating on
u_happy.tsv) plus the other eight: its performance tables.

    python oracle/gen_golden_fairness.py
"""
import glob
import json
import logging
import os
import shutil
import sys
import tempfile
import time
import zlib
from types import SimpleNamespace

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs  # noqa: E402
from oracle.gen_golden_metrics import _as_array, _frame  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")


def entries(user, item, names=("Happiness", "Popularity")):
    """All nine metrics over a user file and an item file (None: the entry names no file)."""
    def mad(m, f, name):
        return {"metric": m, **({"clustering_name": name, "clustering_file": f} if f else {})}
    out = [mad("UserMADrating", user, names[0]), mad("UserMADranking", user, names[0]),
           mad("ItemMADrating", item, names[1]), mad("ItemMADranking", item, names[1])]
    for m in ("REO", "RSP"):
        out.append({"metric": m, **({"clustering_name": names[1], "clustering_file": item} if item else {})})
    for m in ("BiasDisparityBR", "BiasDisparityBS", "BiasDisparityBD"):
        e = {"metric": m}
        if user:
            e.update(user_clustering_name=names[0], user_clustering_file=user)
        if item:
            e.update(item_clustering_name=names[1], item_clustering_file=item)
        out.append(e)
    return out


def config(top_k, cutoffs, thr, complex_metrics):
    return SimpleNamespace(config_test=True, align_side_with_train=False, top_k=top_k,
                           evaluation=SimpleNamespace(simple_metrics=["nDCG"], relevance_threshold=thr,
                                                      paired_ttest=False, cutoffs=cutoffs,
                                                      complex_metrics=complex_metrics))


def lists(g, data, top_k, repeat_every=5, short_every=7, empty_user=None):
    """Popularity-skewed lists with float scores: distinct unrated items, but every `repeat_every`-th user's list is
    drawn with replacement (repeated items, as Random makes them); some lists are short, one may be empty."""
    n_items = data.num_items
    pop = np.asarray(data.sp_i_train.sum(axis=0)).ravel() + 1.0
    p = pop / pop.sum()
    recs = {}
    for pu, u in enumerate(data.users):
        seen = set(data.i_train_dict[pu])
        if repeat_every and pu % repeat_every == 2:
            cand = [int(i) for i in g.choice(n_items, size=top_k, replace=True, p=p)]
        else:
            cand = [i for i in g.choice(n_items, size=min(n_items, 4 * top_k), replace=False, p=p) if i not in seen]
        n = top_k
        if short_every and pu % short_every == 3:
            n = int(g.integers(1, top_k))
        if u == empty_user:
            n = 0
        scores = np.sort(g.normal(3.0, 1.0, size=n))[::-1]
        recs[u] = [(data.private_items[i], float(s)) for i, s in zip(cand[:n], scores)]
    return recs


def scores_array(data, recs, top_k):
    a = np.zeros((data.num_users, top_k))
    for u, lst in recs.items():
        a[data.public_users[u], :len(lst)] = [s for _, s in lst]
    return a


def frames(seed, n_users, n_items):
    g = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.9
    pop /= pop.sum()
    tr, va, te = [], [], []
    for u in range(n_users):
        uid = 7 + 3 * u
        its = 1000 + 5 * g.choice(n_items + 15, size=int(g.integers(6, 30)), replace=False,
                                  p=np.r_[pop * 0.9, np.full(15, 0.1 / 15)])
        rat = g.integers(1, 6, size=its.size).astype(np.float64)
        if u % 11 == 5:
            rat[:] = np.minimum(rat, 2.0)
        n_tr = max(3, int(0.6 * its.size))
        n_va = (its.size - n_tr) // 2
        tr += [(uid, i, r) for i, r in zip(its[:n_tr], rat[:n_tr])]
        if u % 13 != 2:
            va += [(uid, i, r) for i, r in zip(its[n_tr:n_tr + n_va], rat[n_tr:n_tr + n_va])]
        if u % 17 != 4:
            te += [(uid, i, r) for i, r in zip(its[n_tr + n_va:], rat[n_tr + n_va:])]
    tr, va, te = (np.array(x) for x in (tr, va, te))
    g.shuffle(tr); g.shuffle(va); g.shuffle(te)
    return g, tr, va, te


def user_file(g, n_users, n_clusters, empty_cluster=False):
    """Most dataset users (every 9th is missing) and a few ids the dataset lacks; with empty_cluster the last cluster
    holds only ids the dataset lacks."""
    ids = [7 + 3 * u for u in range(n_users) if u % 9 != 4] + [100000 + j for j in range(6)]
    real = n_clusters - 1 if empty_cluster else n_clusters
    labels = [int(g.integers(0, real)) for _ in ids]
    labels[:real] = range(real)
    if empty_cluster:
        labels[-3:] = [n_clusters - 1] * 3
    return np.array(ids, np.int64), np.array(labels, np.int64)


def item_file(g, n_items, n_clusters):
    """Most catalogue and test-only item ids (every 7th is missing) and ids outside the catalogue."""
    ids = [1000 + 5 * i for i in range(n_items + 15) if i % 7 != 3] + [900000 + j for j in range(5)]
    labels = g.integers(0, n_clusters, size=len(ids))
    labels[:n_clusters] = np.arange(n_clusters)
    return np.array(ids, np.int64), labels.astype(np.int64)


def write(path, ids, labels):
    pd.DataFrame({0: ids, 1: labels}).to_csv(path, sep="\t", header=False, index=False)


def evaluate(data, recs, cutoffs):
    """The reference Evaluator's (keys in order, values[cutoff][split][key])."""
    from elliot.evaluation.evaluator import Evaluator
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    res = ev.eval((recs, recs))
    keys = [m for m in res[cutoffs[0]]["test_results"] if m != "nDCG"]
    vals = np.array([[[float(res[k][s][m]) for m in keys] for s in ("val_results", "test_results")] for k in cutoffs])
    return keys, vals


def make_case(tmp, seed, n_users, n_items, thr, top_k, n_ucl, n_icl, empty=False, empty_cluster=False):
    import elliot.dataset.dataset as ds
    g, tr, va, te = frames(seed, n_users, n_items)
    out = dict(train=tr, val=va, test=te, thr=thr, top_k=top_k)
    uf = itf = None
    if n_ucl:
        out["ufile_ids"], out["ufile_labels"] = user_file(g, n_users, n_ucl, empty_cluster)
        uf = os.path.join(tmp, f"u_{seed}.tsv")
        write(uf, out["ufile_ids"], out["ufile_labels"])
    if n_icl:
        out["ifile_ids"], out["ifile_labels"] = item_file(g, n_items, n_icl)
        itf = os.path.join(tmp, f"i_{seed}.tsv")
        write(itf, out["ifile_ids"], out["ifile_labels"])
    spec = entries(uf, itf)
    cutoffs = sorted({1, 5, 10, top_k})
    data = ds.DataSet(config(top_k, cutoffs, thr, spec), (_frame(tr), _frame(va), _frame(te)), SimpleNamespace())
    empty_user = data.users[[pu for pu in range(data.num_users) if data.test_dict[data.users[pu]]][0]] if empty else None
    recs = lists(g, data, top_k, empty_user=empty_user)
    keys, vals = evaluate(data, recs, cutoffs)
    placeholder = json.dumps(entries("{ufile}" if uf else None, "{ifile}" if itf else None))
    out.update(entries=placeholder, cutoffs=np.array(cutoffs), keys=np.array(keys), values=vals,
               users=np.array(data.users, np.int64), items=np.array(data.items, np.int64),
               rec_idx=_as_array(data, recs, top_k), rec_scores=scores_array(data, recs, top_k))
    return out


def make_cases():
    tmp = tempfile.mkdtemp(prefix="fairness_cases_")
    try:
        cases = {"a": make_case(tmp, 21, 220, 160, 0, 20, 2, 4),
                 "b": make_case(tmp, 22, 260, 200, 3, 15, 3, 1, empty_cluster=True),
                 "c": make_case(tmp, 23, 180, 120, 3, 10, 0, 0, empty=True),
                 "d": make_case(tmp, 24, 240, 420, 3, 20, 2, 300)}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    flat = {f"{c}_{k}": v for c, d in cases.items() for k, v in d.items()}
    np.savez_compressed(os.path.join(OUT, "fairness_cases.npz"), cases=np.array(sorted(cases)), **flat)
    for c, d in cases.items():
        v = d["values"][-1, 1]
        print(c, len(d["keys"]), "keys;", int(np.isnan(v).sum()), "NaN,", int(np.isinf(v).sum()), "inf", flush=True)


def ref_file(name):
    return np.loadtxt(os.path.join(ref_stubs.REF, "data", "movielens_1m", name), dtype=np.int64, delimiter="\t")


def c1_split():
    import elliot.dataset.dataset as ds  # noqa: F401
    from elliot.splitter.base_splitter import Splitter
    from elliot_b200 import synth_c1
    with tempfile.TemporaryDirectory() as tmp:
        tsv = os.path.join(tmp, "dataset.tsv")
        checksum = synth_c1.write_tsv(tsv)
        df = pd.read_csv(tsv, sep="\t", header=None, names=["userId", "itemId", "rating", "timestamp"])
    ns = SimpleNamespace(test_splitting=SimpleNamespace(strategy="random_subsampling", test_ratio=0.2))
    (train, test), = Splitter(df, ns, 42).process_splitting()
    return checksum, train, test


C1_LIST_SEED = 2025


def c1_lists(data, top_k):
    """The C1 golden's lists: (recs dict, private-id array, score array).  They depend only on the dataset's train
    matrix and ids, so any DataSet with the reference's fields and ids draws the same ones."""
    recs = lists(np.random.default_rng(C1_LIST_SEED), data, top_k, repeat_every=0, short_every=0)
    return recs, _as_array(data, recs, top_k), scores_array(data, recs, top_k)


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def make_c1():
    import elliot.dataset.dataset as ds
    from elliot.evaluation.evaluator import Evaluator
    u_happy, i_pop = ref_file("u_happy.tsv"), ref_file("i_pop.tsv")
    tmp = tempfile.mkdtemp(prefix="fairness_c1_")
    try:
        uf, itf = os.path.join(tmp, "u_happy.tsv"), os.path.join(tmp, "i_pop.tsv")
        write(uf, u_happy[:, 0], u_happy[:, 1]); write(itf, i_pop[:, 0], i_pop[:, 1])
        checksum, train, test = c1_split()
        top_k, cutoffs = 20, [5, 10, 20]
        data = ds.DataSet(config(top_k, cutoffs, 0, entries(uf, itf)), (train, test), SimpleNamespace())
        recs, rec_idx, rec_scores = c1_lists(data, top_k)
        ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
        t0 = time.perf_counter()
        res = ev.eval((recs, recs))
        dt = time.perf_counter() - t0
        keys = [m for m in res[20]["test_results"] if m != "nDCG"]
        vals = np.array([[float(res[k]["test_results"][m]) for m in keys] for k in cutoffs])
        table = run_c1(tmp, uf, itf)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(os.path.join(OUT, "fairness_c1.npz"), checksum=np.uint64(checksum), top_k=top_k,
                        cutoffs=np.array(cutoffs), entries=json.dumps(entries("{ufile}", "{ifile}")),
                        u_happy=u_happy, i_pop=i_pop, users=np.array(data.users, np.int64),
                        items=np.array(data.items, np.int64), rec_idx_crc=crc(rec_idx), rec_scores_crc=crc(rec_scores),
                        keys=np.array(keys), values=vals,
                        reference_seconds=dt, **table)
    print("c1", len(keys), "keys", f"{dt:.1f} s", flush=True)


RUN_CUTOFFS = (5, 10)


def run_yaml(tsv, out_dir, extra=""):
    """The C1 MostPop experiment with the advanced configuration's complex entry and the other eight; the clustering
    files sit in ../data/movielens_1m/ from the config's folder."""
    from elliot_b200 import synth_c1
    return synth_c1.experiment_yaml(tsv, out_dir, "MostPop", "", extra=extra, metrics=("nDCG", "HR"),
                                    cutoffs=RUN_CUTOFFS, complex_metrics=run_entries())


def run_entries():
    adv = {"metric": "UserMADrating", "clustering_name": "Happiness", "clustering_file": "../data/movielens_1m/u_happy.tsv"}
    rest = [e for e in entries("../data/movielens_1m/u_happy.tsv", "../data/{0}/i_pop.tsv") if e["metric"] != "UserMADrating"]
    return [adv] + rest


def run_c1(tmp, uf, itf):
    """The reference's run_experiment with run_yaml; returns its performance tables (header and rows per cutoff)."""
    from elliot.run import run_experiment
    from elliot_b200 import synth_c1
    cfg_dir = os.path.join(tmp, "cfg")
    data_dir = os.path.join(tmp, "data", "movielens_1m")
    os.makedirs(cfg_dir); os.makedirs(data_dir)
    shutil.copy(uf, data_dir); shutil.copy(itf, data_dir)
    os.makedirs(os.path.join(tmp, "data", "c1_synth")); shutil.copy(itf, os.path.join(tmp, "data", "c1_synth"))
    tsv = os.path.join(tmp, "dataset.tsv")
    synth_c1.write_tsv(tsv)
    out_dir = os.path.join(tmp, "out")
    logcfg = ref_stubs.write_logger_config(os.path.join(tmp, "logger_config.yml"))
    cfg = os.path.join(cfg_dir, "cfg.yml")
    with open(cfg, "w") as fh:
        fh.write(run_yaml(tsv, out_dir, extra=f"  path_logger_config: {logcfg}\n"))
    t0 = time.time()
    run_experiment(cfg)
    print(f"c1 run_experiment {time.time() - t0:.1f} s", flush=True)
    out = {}
    for k in RUN_CUTOFFS:
        f, = glob.glob(os.path.join(out_dir, "performance", f"rec_cutoff_{k}_*.tsv"))
        df = pd.read_csv(f, sep="\t")
        out[f"run_columns_{k}"] = np.array(df.columns.tolist(), dtype=str)
        out[f"run_values_{k}"] = df.iloc[:, 1:].to_numpy(np.float64)
        out[f"run_models_{k}"] = df.iloc[:, 0].to_numpy().astype(str)
    return out


if __name__ == "__main__":
    ref_stubs.install()
    logging.disable(logging.CRITICAL)
    import warnings
    warnings.simplefilter("ignore")
    if "--skip-cases" not in sys.argv:
        make_cases()
    if "--skip-c1" not in sys.argv:
        make_c1()
