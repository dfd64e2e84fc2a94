"""What the MostPop / Random tests share: the golden cases of tests/golden/unpersonalized_cases.npz loaded into the
mirror's DataSet, and the reference's dicts rebuilt from their flat arrays."""
import os
from types import SimpleNamespace

import numpy as np
import pandas as pd

from elliot_b200.dataset import DataSet

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_G = np.load(os.path.join(GOLD, "unpersonalized_cases.npz"))
CASES = _G["cases"].tolist()
RANDOM = [c for c in CASES if c.startswith("random_")]
CUTOFFS = [5, 10]


def case(c):
    return {k[len(c) + 1:]: _G[k] for k in _G.files if k.startswith(c + "_")}


def frame(a):
    a = np.asarray(a, np.float64).reshape(-1, 3)
    return pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})


def data_of(g):
    """The mirror's DataSet on the case's frames (top_k = k, cutoffs 5 and 10); its ids must be the reference's."""
    cfg = SimpleNamespace(config_test=True, top_k=int(g["k"]),
                          evaluation=SimpleNamespace(simple_metrics=g["metrics"].tolist(), relevance_threshold=0,
                                                     paired_ttest=False, cutoffs=CUTOFFS))
    data = DataSet(cfg, (frame(g["train"]), frame(g["test"])))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    return data


def golden_dict(g, call=0):
    """The reference's {key: [(public item, int score)]} of one call, in its key order."""
    keys, lens, items, scores = (g[f"{n}_{call}"].tolist() for n in ("keys", "lens", "items", "scores"))
    out, at = {}, 0
    for key, n in zip(keys, lens):
        out[key] = list(zip(items[at:at + n], scores[at:at + n]))
        at += n
    return out


def same_dict(a, b):
    """Equal dicts in the same key order, with int scores on both sides."""
    return (list(a) == list(b) and a == b
            and all(type(s) is int for d in (a, b) for lst in d.values() for _, s in lst))


def train_csr(data):
    m = data.sp_i_train.tocsr()
    m.sort_indices()
    return m.indptr.astype(np.int64), m.indices.astype(np.int64)
