"""The fairness goldens (tests/golden/fairness_*.npz, minted by oracle/gen_golden_fairness.py) as the mirror's DataSet
and Evaluator: the clustering tables stored in the npz are written back to files and the entries point at them."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pandas as pd

from elliot_b200.dataset import DataSet

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def frame(a):
    a = np.asarray(a, np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})


def config(top_k, cutoffs, thr, complex_metrics, simple=("nDCG",)):
    return SimpleNamespace(config_test=False, top_k=top_k,
                           evaluation=SimpleNamespace(simple_metrics=list(simple), relevance_threshold=thr,
                                                      paired_ttest=False, cutoffs=list(cutoffs),
                                                      complex_metrics=complex_metrics))


def load_cases():
    g = np.load(os.path.join(GOLD, "fairness_cases.npz"))
    return {c: {k[len(c) + 1:]: g[k] for k in g.files if k.startswith(c + "_")} for c in g["cases"].tolist()}


CASES = load_cases()


def write_file(path, ids, labels):
    pd.DataFrame({0: ids, 1: labels}).to_csv(path, sep="\t", header=False, index=False)
    return path


def entries_of(g, tmp, ukey="ufile", ikey="ifile"):
    """The case's complex_metrics entries with its clustering tables written under tmp."""
    files = {}
    for key, name in ((ukey, "users"), (ikey, "items")):
        if f"{key}_ids" in g:
            files[key] = write_file(os.path.join(str(tmp), f"{name}.tsv"), g[f"{key}_ids"], g[f"{key}_labels"])
    text = str(g["entries"])
    for key, path in files.items():
        text = text.replace("{" + key + "}", path)
    return json.loads(text)


def case_evaluator(c, tmp, simple=("nDCG",)):
    from elliot_b200.evaluation import Evaluator
    g = CASES[c]
    data = DataSet(config(int(g["top_k"]), g["cutoffs"].tolist(), float(g["thr"]), entries_of(g, tmp), simple),
                   (frame(g["train"]), frame(g["val"]), frame(g["test"])))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    return g, data, Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))


def as_recs(data, idx, scores):
    """{public user: [(public item, score)]} of private-id and score arrays (-1 ends a list)."""
    out = {}
    for pu, row in enumerate(idx):
        n = int(np.argmax(row < 0)) if (row < 0).any() else len(row)
        out[data.users[pu]] = [(data.items[i], float(s)) for i, s in zip(row[:n].tolist(), scores[pu, :n].tolist())]
    return out


def assert_matches(got, keys, want, what, rtol=1e-12):
    """Same keys in the same order; values to rtol (1e-12) relative; NaN and inf where the reference has them."""
    assert list(got) == list(keys), what
    g = np.array([got[k] for k in keys], np.float64)
    w = np.asarray(want, np.float64)
    np.testing.assert_array_equal(np.isnan(g), np.isnan(w), err_msg=str(what))
    np.testing.assert_array_equal(np.isinf(g) * np.sign(g), np.isinf(w) * np.sign(w), err_msg=str(what))
    ok = np.isfinite(w)
    np.testing.assert_allclose(g[ok], w[ok], rtol=rtol, atol=1e-15, err_msg=str(what))


def fairness_part(res):
    return {k: v for k, v in res.items() if k != "nDCG"}
