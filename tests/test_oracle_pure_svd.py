"""The fp64 PureSVD restatement (oracle/pure_svd.py) against the reference's goldens: singular values within 1e-5 of the
largest, scores within 1e-5 max |P|, the orientation of every determined user-side column, and the reference's top-k
lists at every isolated rank; and its pivoted CholeskyQR on rank-deficient blocks."""
import os

import numpy as np
import pytest

from oracle import pure_svd as opsvd

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_G = dict(np.load(os.path.join(GOLD, "pure_svd_cases.npz")))


def case(name):
    return {"R": _G[f"{name}_R"].astype(np.float64), "s": _G[f"{name}_s"], "user_vec": _G[f"{name}_user_vec"],
            "item_vec": _G[f"{name}_item_vec"], "topk_idx": _G[f"{name}_topk_idx"]}


@pytest.mark.parametrize("name", list(_G["cases"]))
def test_oracle_matches_the_reference(name):
    c = case(name)
    user, item, s = opsvd.fit(c["R"], int(_G[f"{name}_factors"]), int(_G["seed"]))
    assert user.shape == c["user_vec"].shape and item.shape == c["item_vec"].shape
    err, n_iso = opsvd.check_against(c, user, item, s)
    if int(_G[f"{name}_factors"]) < min(c["R"].shape):     # a full-rank fit scores every unseen item ~0: no isolated rank
        assert n_iso > 0.5 * c["topk_idx"].size, n_iso


@pytest.mark.parametrize("shape,rank", [((60, 40), 39), ((200, 45), 12), ((30, 45), 30)])
def test_pivoted_cholesky_qr_keeps_the_rank(shape, rank):
    g = np.random.default_rng(rank)
    X = g.standard_normal((shape[0], rank)) @ g.standard_normal((rank, shape[1]))
    Y = opsvd.orth(X)
    nz = np.abs(Y).max(0) > 0
    assert nz.sum() == rank
    assert np.abs(Y[:, nz].T @ Y[:, nz] - np.eye(rank)).max() < 1e-12
    # same column space: projecting X onto it loses nothing
    assert np.abs(Y @ (Y.T @ X) - X).max() < 1e-10 * np.abs(X).max()


def test_goldens_record_the_sklearn_version():
    assert str(_G["sklearn_version"])
    assert str(np.load(os.path.join(GOLD, "pure_svd_c1.npz"))["sklearn_version"])
