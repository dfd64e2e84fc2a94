"""CPU: the fp64 EASE^R restatement (oracle/ease.py) against the reference's own runs (tests/golden/ease_cases.npz, minted
by oracle/gen_golden_ease.py), the C1 golden's shape, and the options the model refuses."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import ease as oease
from oracle.knn import isolated

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden():
    return dict(np.load(os.path.join(GOLD, "ease_cases.npz")))


CASES = list(_golden()["cases"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    g = _golden()
    R = g[f"{name}_R"].astype(np.float64)
    k = int(g["topk"])
    _, P, oi, ov = oease.run(R, float(g[f"{name}_l2_norm"]), k + 1)
    ref = g[f"{name}_preds"].astype(np.float64)
    assert np.abs(P - ref).max() <= 1e-5 * np.abs(ref).max(), name
    ti, tv = g[f"{name}_topk_idx"], g[f"{name}_topk_val"]
    assert np.array_equal(oi[:, :k] >= 0, np.isfinite(tv)), name
    iso = isolated(ov[:, :k], ov[:, k])
    assert iso.mean() > 0.85, (name, iso.mean())
    assert np.array_equal(oi[:, :k][iso], ti[iso]), name


def test_goldens_cover_the_issue_cases():
    g = _golden()
    lams = {float(g[f"{n}_l2_norm"]) for n in CASES}
    assert lams == {1e3, 10.0, 0.3}
    kinds = set()
    for n in CASES:
        R = g[f"{n}_R"].astype(np.float64)
        vals = np.unique(R[R != 0])
        kinds.add("implicit" if np.array_equal(vals, [1.0]) else "half" if np.any(vals != np.round(vals)) else "int")
        assert np.any(R.sum(0) == 0), "a cold item"
        assert np.any(R.sum(1) == 0), "a user without ratings"
        assert np.array_equal(R[:, 0], R[:, 1]), "a duplicated item"
    assert kinds == {"int", "implicit", "half"}
    assert max(g[f"{n}_R"].shape[1] for n in CASES) > 4 * 64, "the blocked inverse must span several panels"


def test_explicit_normal_matrix_is_indefinite():
    """Why the inverse is an LU-type elimination: with ratings 1-5 the diagonal count + l2_norm is below sum r^2, and the
    matrix has negative eigenvalues; with implicit ones it is positive definite."""
    g = _golden()
    G = oease.normal_matrix(g["int_l10_R"].astype(np.float64), 10.0)
    assert np.linalg.eigvalsh(G)[0] < 0
    G = oease.normal_matrix(g["implicit_l0.3_R"].astype(np.float64), 0.3)
    assert np.linalg.eigvalsh(G)[0] > 0


def test_diagonal_is_the_float32_sum():
    R = np.zeros((3, 2))
    R[0, 0] = R[1, 0] = 1.0
    G = oease.normal_matrix(R, 0.3)
    assert G[0, 0] == float(np.float32(2.3)) and G[0, 0] != 2.3
    assert G[1, 1] == float(np.float32(0.3))


def test_c1_golden_is_complete():
    g = dict(np.load(os.path.join(GOLD, "ease_c1.npz")))
    assert str(g["rec_file"]) == "EASER_neighborhood=3706_l2_norm=1000$0.tsv"
    users = np.unique(g["rec_users"])
    assert len(users) == 400 and len(g["rec_items"]) == 400 * 10
    assert g["test_metrics"].shape == (4,)


class _Ns(SimpleNamespace):
    pass


def _make(**block):
    """Build EASER up to the option checks (no device is touched before them)."""
    from elliot_b200.recommender import ease
    ev = _Ns(cutoffs=[10], simple_metrics=["nDCG"], relevance_threshold=0)
    cfg = _Ns(evaluation=ev, top_k=10, path_output_rec_weight="/nonexistent", path_output_rec_result="/nonexistent")
    data = _Ns(config=cfg, num_items=3, num_users=3)
    params = _Ns(meta=_Ns(**block.pop("meta", {})), **block)
    return ease.EASER(data=data, config=cfg, params=params)


@pytest.mark.parametrize("meta", [{"save_weights": True}, {"restore": True}])
def test_weights_io_raises(meta):
    with pytest.raises(NotImplementedError, match="dense prediction matrix"):
        _make(meta=meta)


def test_model_is_registered():
    from elliot_b200 import external, recommender
    assert hasattr(recommender, "EASER")
    assert hasattr(external, "EASER")
