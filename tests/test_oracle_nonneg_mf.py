"""The NonNegMF oracle (oracle/nonneg_mf.py) against the goldens minted from the unmodified reference: mu and every
table of every epoch bit for bit; and the model's name, which follows batch_size like the reference's."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import nonneg_mf as onm

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_G = dict(np.load(os.path.join(GOLD, "nonneg_mf_cases.npz")))
CASES = list(_G["cases"])


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_every_epoch_bit_for_bit(name):
    U, I, F = (int(x) for x in _G[f"{name}_shape"])
    indptr, items, vals = _G[f"{name}_indptr"], _G[f"{name}_items"].astype(np.int64), _G[f"{name}_ratings"]
    lr, reg, seed = float(_G[f"{name}_lr"]), float(_G[f"{name}_reg"]), int(_G[f"{name}_seed"])
    rows = onm.row_of(indptr)
    mu = np.mean(sp.csr_matrix((vals, (rows, items)), dtype="float32", shape=(U, I)))
    assert np.array_equal(_bits(np.float64(mu)), _bits(_G[f"{name}_mu"]))
    P, Q = onm.init_tables(seed, U, I, F)
    assert np.array_equal(_bits(P), _bits(_G[f"{name}_P"][0])) and np.array_equal(_bits(Q), _bits(_G[f"{name}_Q"][0]))
    bu, bi = np.zeros(U), np.zeros(I)
    for e in range(int(_G["epochs"])):
        P, Q, _, _ = onm.epoch(P, Q, bu, bi, mu, indptr, items, vals, lr, reg)
        for key, got in (("P", P), ("Q", Q), ("bu", bu), ("bi", bi)):
            assert np.array_equal(_bits(got), _bits(_G[f"{name}_{key}"][e + 1])), (name, e, key)


def test_goldens_cover_the_edge_rows():
    for name in CASES:
        indptr, items = _G[f"{name}_indptr"], _G[f"{name}_items"]
        I = int(_G[f"{name}_shape"][1])
        assert np.diff(indptr).min() == 1                                  # a one-rating user
        assert np.bincount(items, minlength=I).min() == 1                  # a one-rating item, and no cold item
        assert (_G[f"{name}_topk_idx"] < 0).any()                          # a user with fewer than k candidates
        assert (_G[f"{name}_ratings"] == 0).any()                          # explicit 0 ratings
    assert sorted(int(_G[f"{n}_shape"][2]) for n in CASES) == [1, 10, 33]


class _Ns(SimpleNamespace):
    pass


def _name(monkeypatch, tmp_path, **block):
    """NonNegMF's name for a YAML block, with the device parts replaced (the name needs none of them)."""
    from elliot_b200 import evaluation
    from elliot_b200.recommender import nonneg_mf
    monkeypatch.setattr(nonneg_mf, "cuda_device", lambda params, who: None)
    monkeypatch.setattr(nonneg_mf, "NonNegMFModel", lambda *a, **k: None)
    monkeypatch.setattr(nonneg_mf, "train_csr_of", lambda *a, **k: (None, None, None))
    monkeypatch.setattr(evaluation, "Evaluator", lambda data, params: None)
    ev = _Ns(cutoffs=[10], simple_metrics=["nDCG"], relevance_threshold=0)
    cfg = _Ns(evaluation=ev, top_k=10, path_output_rec_weight=str(tmp_path), path_output_rec_result=str(tmp_path))
    data = _Ns(config=cfg, num_items=3, num_users=2, users=[0, 1], items=[0, 1, 2], transactions=4,
               sp_i_train_ratings=sp.csr_matrix(np.array([[1, 0, 2], [0, 3, 4]], np.float32)))
    params = _Ns(meta=_Ns(), **block)
    return nonneg_mf.NonNegMF(data=data, config=cfg, params=params).name


def test_name_follows_batch_size(monkeypatch, tmp_path):
    assert (_name(monkeypatch, tmp_path, epochs=10, batch_size=512, factors=10, lr=0.001, reg=0.1)
            == "NonNegMF_seed=42_e=10_bs=512_factors=10_lr=0$001_reg=0$1")
    assert _name(monkeypatch, tmp_path, epochs=3, factors=4) == "NonNegMF_seed=42_e=3_bs=4_factors=4_lr=0$001_reg=0$1"
    assert _name(monkeypatch, tmp_path, epochs=3, batch_size=0) == "NonNegMF_seed=42_e=3_bs=4_factors=10_lr=0$001_reg=0$1"


def test_model_is_registered():
    from elliot_b200 import external, recommender
    assert hasattr(recommender, "NonNegMF") and hasattr(external, "NonNegMF")
