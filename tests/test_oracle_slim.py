"""The numpy SLIM restatement (oracle/slim.py) against the reference's goldens (tests/golden/slim_cases.npz, minted by
oracle/gen_golden_slim.py from the unmodified SlimModel and sklearn's ElasticNet): every item's coefficients within
1e-5 of its largest, equal epoch counts, W equal except at ties, scores from the golden's W bit-equal to the
reference's preds, and the top-k lists equal at isolated ranks."""
import os

import numpy as np
import pytest

from oracle import slim as oslim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_G = dict(np.load(os.path.join(ROOT, "tests", "golden", "slim_cases.npz")))


@pytest.mark.parametrize("name", list(_G["cases"]))
def test_oracle_matches_the_reference(name):
    oslim.check_case(_G, name)


def test_xorshift_matches_the_reference_stream():
    s = np.array([oslim.seed_state(42)], np.uint32)
    x = int(s[0])
    for _ in range(50):
        x ^= (x << 13) & 0xffffffff
        x ^= x >> 17
        x ^= (x << 5) & 0xffffffff
        assert int(oslim.xorshift(s)[0]) == x % 2 ** 31


def test_nnz_minus_one_rule_and_empty_columns():
    coef = np.zeros((4, 4), np.float32)
    coef[0, [1, 2, 3]] = [0.5, 0.25, 0.25]          # 3 nonzeros <= neighborhood: the smallest goes, tie -> item 3
    coef[1, [0]] = [1.0]                             # 1 nonzero: nothing kept
    coef[3, [0, 1, 2]] = [0.1, 0.3, 0.2]             # more than neighborhood 2: the 2 largest
    W = oslim.select(coef, 3).toarray()
    assert W[:, 0].tolist() == [0, 0.5, 0.25, 0]
    assert not W[:, 1].any() and not W[:, 2].any()
    assert np.allclose(W[:, 3], [0, 0.3, 0.2, 0])
    assert oslim.select(coef, 2).toarray()[:, 3].tolist() == pytest.approx([0, 0.3, 0.2, 0])


def test_more_items_than_users_is_refused():
    with pytest.raises(ValueError, match="num_items <= num_users"):
        oslim.fit(np.ones((3, 5), np.float32), 0.05, 0.5, 42)


def test_goldens_record_the_solver_version():
    assert str(_G["sklearn_version"])
