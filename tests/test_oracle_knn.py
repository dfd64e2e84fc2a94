"""CPU: the fp64 ItemKNN / UserKNN restatement (oracle/knn.py) against the reference's own runs (tests/golden/*knn*.npz,
minted by oracle/gen_golden_knn.py), and the host-side rules of elliot_b200.recommender.knn."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import knn as oknn
from oracle.knn import isolated

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = [(m, s) for m in ("itemknn", "userknn") for s in ("tiny", "small")]
TAGS = [f"{kind}_{sim}" for kind in ("int", "implicit", "half") for sim in ("cosine", "dot")]


def _ulp4(v):
    return 4 * np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


@pytest.mark.parametrize("model,size", CASES)
def test_oracle_matches_reference_goldens(model, size):
    g = dict(np.load(os.path.join(GOLD, f"{model}_{size}.npz")))
    over, k_nn, k = str(g["over"]), int(g["k_nn"]), int(g["topk"])
    for tag in TAGS:
        R = g[f"{tag}_R"]
        Ru = (R != 0).astype(np.float64) if tag.startswith("implicit") else R
        S = oknn.similarity(oknn.gram(Ru, over), tag.endswith("cosine"))
        oi, ov, _ = oknn.neighbours(S, k_nn + 1)
        ri, rv = g[f"{tag}_nbr_idx"], g[f"{tag}_nbr_val"]
        for r in range(S.shape[0]):
            want = set(ri[r][ri[r] >= 0].tolist())
            got = oi[r, :k_nn]
            got = set(got[got >= 0].tolist())
            # the sets agree wherever the k-th and (k+1)-th similarities are more than 4 fp32 ulp apart
            if oi[r, k_nn] < 0 or ov[r, k_nn - 1] - ov[r, k_nn] > _ulp4(ov[r, k_nn - 1]):
                assert got == want, (tag, r)
            np.testing.assert_allclose(np.sort(rv[r][ri[r] >= 0]), np.sort(ov[r, :len(want)]), rtol=1e-6, atol=1e-7)
        # preds over the reference's own lists (exact ties at rank k_nn may be broken either way)
        P = oknn.preds(Ru, ri, rv, over)
        scale = max(np.abs(g[f"{tag}_preds"]).max(), 1.0)
        assert np.abs(P - g[f"{tag}_preds"]).max() <= 1e-5 * scale, tag
        ti, tv = oknn.topk(P, R != 0, k + 1)
        gv = g[f"{tag}_topk_val"]
        iso = isolated(gv, tv[:, k])
        assert np.array_equal(ti[:, :k][iso], g[f"{tag}_topk_idx"][iso]), tag
        assert np.array_equal(ti[:, :k] >= 0, np.isfinite(gv)), tag


def test_exactness_rule():
    from elliot_b200.recommender.knn import exactness_scale
    assert exactness_scale(np.array([1, 2, 3, 4, 5], np.float32)) == 0
    assert exactness_scale(np.ones(7, np.float32)) == 0
    assert exactness_scale(np.array([0.5, 1.5, 4.5, 5], np.float32)) == 1
    assert exactness_scale(np.array([0.25, 3], np.float32)) == 2
    with pytest.raises(ValueError):
        exactness_scale(np.array([0.3, 1], np.float32))
    with pytest.raises(ValueError):
        exactness_scale(np.array([300, 1], np.float32))


def test_frac_bits_keep_sums_below_2_62():
    from elliot_b200.recommender.knn import frac_bits
    for b in (1e-9, 0.75, 1.0, 5.0, 11500.0, 2.0 ** 40, 3.0 ** 30):
        f = frac_bits(b)
        assert b * 2.0 ** f < 2.0 ** 61 <= 2 * b * 2.0 ** f * 2
    assert frac_bits(0.0) == 0


class _Ns(SimpleNamespace):
    pass


def _make(cls, **block):
    """Build ItemKNN / UserKNN up to the option checks (no device is touched before them)."""
    from elliot_b200.recommender import knn
    ev = _Ns(cutoffs=[10], simple_metrics=["nDCG"], relevance_threshold=0)
    cfg = _Ns(evaluation=ev, top_k=10, path_output_rec_weight="/nonexistent", path_output_rec_result="/nonexistent")
    data = _Ns(config=cfg, num_items=3, num_users=3)
    params = _Ns(meta=_Ns(**block.pop("meta", {})), **block)
    return getattr(knn, cls)(data=data, config=cfg, params=params)


@pytest.mark.parametrize("cls", ["ItemKNN", "UserKNN"])
@pytest.mark.parametrize("block", [{"implementation": "aiolli"}, {"similarity": "euclidean"}, {"similarity": "jaccard"},
                                   {"meta": {"save_weights": True}}, {"meta": {"restore": True}}])
def test_unsupported_options_raise(cls, block):
    with pytest.raises(NotImplementedError):
        _make(cls, **block)
