"""CPU: the fp64 iALS / WRMF restatement (oracle/als.py) against the reference's own runs (tests/golden/als_cases.npz,
minted by oracle/gen_golden_als.py), the host-side confidences of elliot_b200.recommender.als, and the options the models
refuse."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import als as oals

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden():
    return dict(np.load(os.path.join(GOLD, "als_cases.npz")))


def _case(g, name):
    d, alpha, eps, reg = g[f"{name}_hp"].tolist()
    kind = "iALS" if name.startswith("ials") else "WRMF"
    return kind, int(d), alpha, (1.0 if np.isnan(eps) else eps), reg, str(g[f"{name}_scaling"])


CASES = list(_golden()["cases"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    g = _golden()
    kind, d, alpha, eps, reg, scaling = _case(g, name)
    R = g[f"{name}_R"].astype(np.float64)
    out, _ = oals.train(kind, sp.csr_matrix(R), g[f"{name}_X0"], g[f"{name}_Y0"], int(g["epochs"]), alpha, reg, eps,
                        scaling if kind == "iALS" else "linear")
    for e, (X, Y) in enumerate(out):
        assert np.abs(X - g[f"{name}_X"][e]).max() <= 1e-12, (name, e)
        assert np.abs(Y - g[f"{name}_Y"][e]).max() <= 1e-12, (name, e)
    idx, _ = oals.topk(out[-1][0], out[-1][1], R != 0, int(g["topk"]))
    assert np.array_equal(idx, g[f"{name}_topk_idx"]), name


@pytest.mark.parametrize("name", CASES)
def test_confidences_bit_equal_to_the_reference(name):
    """The reference's float32 C (iALS: 1 + alpha r or the log form; WRMF: alpha r) is reproduced bit for bit by the
    oracle and by the model's host code, and w / c follow from it as the reference promotes them."""
    from elliot_b200.recommender import als
    g = _golden()
    kind, d, alpha, eps, reg, scaling = _case(g, name)
    m = sp.csr_matrix(g[f"{name}_R"].astype(np.float32))
    m.sort_indices()
    ref = g[f"{name}_conf"]
    assert ref.dtype == np.float32
    if kind == "iALS":
        for w, c in (oals.ials_confidences(m.data, alpha, eps, scaling), als.ials_confidences(m.data, alpha, eps, scaling)):
            assert np.array_equal(c, ref.astype(np.float64))
            assert np.array_equal(w, (ref - np.float32(1)).astype(np.float64))
    else:
        a = int(alpha) if float(alpha).is_integer() else alpha
        for w, c in (oals.wrmf_confidences(m.data, a), als.wrmf_confidences(m, a)):
            assert np.array_equal(w, ref.astype(np.float64))
            assert np.array_equal(c, ref.astype(np.float64) + 1.0)


def test_non_integer_alpha_makes_float32_confidences_differ_from_fp64():
    g = _golden()
    kind, d, alpha, eps, reg, scaling = _case(g, "ials_lin_d10")
    assert not float(alpha).is_integer()
    assert not np.array_equal(g["ials_lin_d10_conf"].astype(np.float64), 1.0 + alpha * np.ones(1))


def test_goldens_cover_the_issue_cases():
    g = _golden()
    ds = {_case(g, n)[1] for n in CASES}
    assert ds == {1, 10, 33}
    assert {_case(g, n)[5] for n in CASES if n.startswith("ials")} >= {"linear", "log"}
    for n in CASES:
        R = g[f"{n}_R"]
        cold = np.flatnonzero(R.sum(0) == 0)
        assert cold.size >= 1
        if n.startswith("ials"):              # cold items keep their initial rows
            assert np.array_equal(g[f"{n}_Y"][-1][cold], g[f"{n}_Y0"][cold])
        else:                                 # WRMF solves them to 0
            assert np.all(g[f"{n}_Y"][-1][cold] == 0)


class _Ns(SimpleNamespace):
    pass


def _make(cls, **block):
    """Build iALS / WRMF up to the option checks (no device is touched before them)."""
    from elliot_b200.recommender import als
    ev = _Ns(cutoffs=[10], simple_metrics=["nDCG"], relevance_threshold=0)
    cfg = _Ns(evaluation=ev, top_k=10, path_output_rec_weight="/nonexistent", path_output_rec_result="/nonexistent")
    data = _Ns(config=cfg, num_items=3, num_users=3)
    params = _Ns(meta=_Ns(**block.pop("meta", {})), **block)
    return getattr(als, cls)(data=data, config=cfg, params=params)


@pytest.mark.parametrize("cls", ["iALS", "WRMF"])
def test_too_many_factors_raise(cls):
    with pytest.raises(ValueError, match="200"):
        _make(cls, factors=201)
    with pytest.raises(ValueError, match="factors"):
        _make(cls, factors=0)


@pytest.mark.parametrize("cls", ["iALS", "WRMF"])
@pytest.mark.parametrize("meta", [{"save_weights": True}, {"restore": True}])
def test_weights_io_raises(cls, meta):
    with pytest.raises(NotImplementedError, match="dense prediction matrix"):
        _make(cls, meta=meta)


def test_models_are_registered():
    from elliot_b200 import external, recommender
    for name in ("iALS", "WRMF"):
        assert hasattr(recommender, name)
        assert hasattr(external, name)
