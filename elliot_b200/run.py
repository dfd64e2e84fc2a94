"""run_experiment(config_path): drives the GPU models from an Elliot YAML file.

Mirrors the call contract of elliot/run.py:39-148 for the slice the hot path needs: read the
YAML (namespace_model.py:64-241 keys), load + split the data (dataset.py:29-161,
base_splitter.py:62-111,256-274 — same legacy-numpy split stream, so identical splits for the
same file and seed), resolve each model key (built-in name or `external.<Class>` through
`external_models_path`, run.py:67-75), run `model.train()` once per model (the
ModelCoordinator.single path, model_coordinator.py:83-117) and write the performance table.
Out of scope: hyperopt search spaces, prefiltering, side information, statistical tests.
"""
import importlib
import importlib.util
import json
import math
import os
import re
from types import SimpleNamespace

import numpy as np
import pandas as pd
import yaml

from .dataset import DataSet

COLS = ["userId", "itemId", "rating", "timestamp"]


def _abs(cfg_dir, p):
    return p if os.path.isabs(p) else os.path.abspath(os.path.join(cfg_dir, p))


# a word, a dot and a word somewhere in the value, after a first character that is not a digit: a file name
_FILE_LIKE = re.compile(r"[\D][\w-]+\.[\w-]+")


def resolve_param(cfg_dir, value, dataset):
    """A complex metric parameter as the reference's namespace builder reads it: strings get `{0}` = the dataset name;
    an absolute path is kept (normalised), a relative one starting with `.` or looking like a file name is taken from
    the config file's folder, any other string is a plain value.  Non-strings are returned as they are."""
    if not isinstance(value, str):
        return value
    value = value.format(dataset)
    if os.path.isabs(value):
        return os.path.abspath(value)
    if value.startswith(".") or _FILE_LIKE.search(value):
        return os.path.abspath(os.path.join(cfg_dir, value))
    return value


def _read(path, binarize):
    df = pd.read_csv(path, sep="\t", header=None, names=COLS)
    if df["timestamp"].isna().all():
        df = df.drop(columns=["timestamp"]).reset_index(drop=True)
    if binarize or df["rating"].isna().all():
        df["rating"] = 1
    return df


def split_random_subsampling(df, ratio, seed, folds=1):
    """base_splitter.py:62-72 + 256-274: np.random.seed(seed); users in sorted groupby order;
    per user a [0]*train + [1]*test flag list shuffled with the legacy global stream."""
    np.random.seed(seed)
    out = []
    groups = [(name, grp.index.to_numpy()) for name, grp in df.groupby("userId")]
    for _ in range(folds):
        flag = np.zeros(len(df), dtype=np.int8)
        for _, index in groups:
            n = len(index)
            n_train = int(math.floor(n * (1 - ratio)))
            lst = [0] * n_train + [1] * (n - n_train)
            np.random.shuffle(lst)
            flag[index] = lst
        out.append((df[flag == 0].reset_index(drop=True), df[flag == 1].reset_index(drop=True)))
    return out


def build_base_config(path):
    cfg_dir = os.path.dirname(os.path.abspath(path))
    raw = yaml.safe_load(open(path))["experiment"]
    name = raw["dataset"]
    ev = raw.get("evaluation", {})
    res = lambda kind, sub: _abs(cfg_dir, raw.get(kind, os.path.join("..", "results", "{0}", sub)).format(name))
    base = SimpleNamespace(
        dataset=name, top_k=raw.get("top_k", 10), random_seed=raw.get("random_seed", 42),
        binarize=raw.get("binarize", False), config_test=False, align_side_with_train=False,
        path_output_rec_result=res("path_output_rec_result", "recs"),
        path_output_rec_weight=res("path_output_rec_weight", "weights"),
        path_output_rec_performance=res("path_output_rec_performance", "performance"),
        external_models_path=raw.get("external_models_path"),
        evaluation=SimpleNamespace(simple_metrics=ev.get("simple_metrics", ["nDCG"]),
                                   relevance_threshold=ev.get("relevance_threshold", 0),
                                   paired_ttest=False, wilcoxon_test=False,
                                   complex_metrics=[{k: resolve_param(cfg_dir, v, name) for k, v in entry.items()}
                                                    for entry in ev.get("complex_metrics") or []],
                                   **({"cutoffs": ev["cutoffs"]} if "cutoffs" in ev else {})),
        data_config=SimpleNamespace(**raw["data_config"]),
        splitting=raw.get("splitting"),
    )
    if base.external_models_path:
        base.external_models_path = _abs(cfg_dir, base.external_models_path)
    for k in ("dataset_path", "train_path", "test_path", "validation_path"):
        if hasattr(base.data_config, k):
            setattr(base.data_config, k, _abs(cfg_dir, getattr(base.data_config, k)))
    if "negative_sampling" in raw:
        raise NotImplementedError("evaluation-time negative sampling is outside this build's scope")
    for d in (base.path_output_rec_result, base.path_output_rec_weight, base.path_output_rec_performance):
        os.makedirs(d, exist_ok=True)
    return base, raw.get("models", {})


def load_folds(base):
    dc = base.data_config
    if dc.strategy == "fixed":
        tr = _read(dc.train_path, base.binarize); te = _read(dc.test_path, base.binarize)
        if getattr(dc, "validation_path", None):
            return [(tr, _read(dc.validation_path, base.binarize), te)]
        return [(tr, te)]
    if dc.strategy == "dataset":
        df = _read(dc.dataset_path, base.binarize)
        ts = (base.splitting or {}).get("test_splitting")
        if not ts or ts.get("strategy") != "random_subsampling" or "test_ratio" not in ts:
            raise NotImplementedError("only test_splitting: {strategy: random_subsampling, test_ratio} is mirrored")
        if "validation_splitting" in base.splitting:
            raise NotImplementedError("validation_splitting is not mirrored")
        return split_random_subsampling(df, float(ts["test_ratio"]), base.random_seed, int(ts.get("folds", 1)))
    raise Exception("Strategy option not recognized")


def _params_namespace(block):
    block = dict(block or {})
    meta = SimpleNamespace(**block.pop("meta", {}))
    for k, v in block.items():
        if isinstance(v, list):
            if len(v) != 1:
                raise NotImplementedError(f"hyper-parameter search space for '{k}' needs hyperopt (out of scope)")
            block[k] = v[0]
    return SimpleNamespace(meta=meta, **block)


def _resolve(key, base):
    if key.startswith("external."):
        spec = importlib.util.spec_from_file_location("external", base.external_models_path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return getattr(mod, key.split(".", 1)[1])
    return getattr(importlib.import_module("elliot_b200.recommender"), key)


def run_experiment(config_path: str = ""):
    base, models = build_base_config(config_path)
    folds = load_folds(base)
    all_results = []
    for key, block in models.items():
        cls = _resolve(key, base)
        fold_results = []
        for tup in folds:
            data = DataSet(base, tup)
            model = cls(data=data, config=base, params=_params_namespace(block))
            model.train()
            res = model.get_results()
            fold_results.append({"loss": model.get_loss(), "params": {k: v for k, v in model.get_params().items() if k != "meta"},
                                 "val_results": {k: res[k]["val_results"] for k in res},
                                 "test_results": {k: res[k]["test_results"] for k in res},
                                 "name": model.name,
                                 # every evaluated epoch's test metrics (the reference only logs them)
                                 "history": [{k: r[k]["test_results"] for k in r} for r in model._results]})
        best = min(fold_results, key=lambda r: r["loss"])
        all_results.append(best)
    # performance table (result_handler.py:40-81 layout: one row per model, one column per metric)
    for k in sorted({kk for r in all_results for kk in r["test_results"]}):
        rows = [{"model": r["name"], **r["test_results"][k]} for r in all_results]
        pd.DataFrame(rows).to_csv(os.path.join(base.path_output_rec_performance, f"rec_cutoff_{k}.tsv"), sep="\t", index=False)
    with open(os.path.join(base.path_output_rec_performance, "results.json"), "w") as f:
        json.dump(all_results, f, indent=1, default=str)
    return all_results
