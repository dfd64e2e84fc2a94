"""The SlopeOne oracle (oracle/slope_one.py) against the goldens minted from the unmodified reference: `dev` (CRC and
rows), the user means and every recorded score bit for bit, the lists at isolated ranks, and the dict order mattering."""
import os

import numpy as np
import pytest

from oracle import slope_one as oso

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_G = dict(np.load(os.path.join(GOLD, "slope_one_cases.npz")))
CASES = list(_G["cases"])


def _case(name):
    return (int(_G[f"{name}_n_items"]), _G[f"{name}_indptr"], _G[f"{name}_items"].astype(np.int64),
            _G[f"{name}_ratings"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_bit_for_bit(name):
    I, indptr, items, vals = _case(name)
    assert I >= 2048
    F, E = oso.deviations(indptr, items, vals, I)
    dev = oso.reference_dev(E)
    assert oso.crc(dev) == int(_G[f"{name}_dev_crc"])
    rows = _G[f"{name}_dev_rows"]
    assert np.array_equal(dev[rows].view(np.uint64), _G[f"{name}_dev"].view(np.uint64))
    means = oso.user_means(indptr, vals)
    assert np.array_equal(means.view(np.uint64), _G[f"{name}_means"].view(np.uint64))
    P = oso.scores(E, means, indptr, items)
    ti, tv = _G[f"{name}_topk_idx"], _G[f"{name}_topk_val"]
    ok = ti >= 0
    got = np.take_along_axis(P, np.where(ok, ti, 0), 1)
    assert np.array_equal(got[ok].view(np.uint64), tv[ok].view(np.uint64))
    # the lists: the same length, and the same item wherever the rank's value is isolated
    K = int(_G["topk"])
    oi, ov = oso.topk(P, indptr, items, K + 1)
    assert np.array_equal(ok, oi[:, :K] >= 0)
    iso = oso.isolated(ov)[:, :K]
    assert np.array_equal(oi[:, :K][iso], ti[iso])
    assert np.array_equal(ov[:, :K][ok].view(np.uint64), tv[ok].view(np.uint64))    # sorted the same way


def test_the_cases_cover_the_documented_shapes():
    K = int(_G["topk"])
    seen = set()
    for name in CASES:
        I, indptr, items, vals = _case(name)
        lens = np.diff(indptr)
        seen.add("odd width" if I % 8 else "width of 8s")
        if (lens == 1).any():
            seen.add("one-item user")
        if ((I - lens) < K).any():
            seen.add("fewer than k candidates")
        if (vals == 0).any():
            seen.add("explicit 0")
        if np.setdiff1d(np.arange(I), items).size:
            seen.add("cold item")
        if (vals * 2 != np.round(vals * 2)).any() or (vals != np.round(vals)).any():
            seen.add("half stars")
        if np.unique(vals).size == 1:
            seen.add("all equal")
    assert {"odd width", "one-item user", "fewer than k candidates", "explicit 0", "cold item", "half stars",
            "all equal"} <= seen, seen


def test_the_dict_order_changes_some_scores():
    assert sum(int(_G[f"{name}_order_sensitive"]) for name in CASES) > 0
    name = "stars"
    I, indptr, items, vals = _case(name)
    F, E = oso.deviations(indptr, items, vals, I)
    means = oso.user_means(indptr, vals)
    P = oso.scores(E, means, indptr, items)
    Ps = oso.scores(E, means, indptr, oso.sorted_rows(indptr, items, vals)[0])
    cand = np.ones(P.shape, bool)
    cand[np.repeat(np.arange(len(indptr) - 1), np.diff(indptr)), items] = False
    assert int((cand & (P != Ps)).sum()) == int(_G[f"{name}_order_sensitive"])
