"""SlopeOne's host side without a GPU: the dict-order train CSR (the DataSet's grouped arrays and the i_train_dict of any
object with the DataSet's fields give the same rows), and the refusal of ratings outside the exactness class."""
import numpy as np
import pandas as pd
import pytest

from elliot_b200.dataset import DataSet
from elliot_b200.recommender.slope_one import SlopeOneModel, dict_order_csr


class _Fields:
    """Only the DataSet fields a drop-in caller is guaranteed to have."""

    def __init__(self, ds):
        self.users, self.items, self.i_train_dict = ds.users, ds.items, ds.i_train_dict


def _dataset(ratings):
    g = np.random.default_rng(3)
    n = len(ratings)
    tr = pd.DataFrame({"userId": g.integers(1, 30, n), "itemId": g.integers(1, 80, n), "rating": ratings,
                       "timestamp": np.arange(n)})
    return DataSet(None, (tr, tr.iloc[:5]))


def test_dict_order_csr_follows_i_train_dict():
    ds = _dataset(np.random.default_rng(4).integers(0, 6, 600).astype(float))
    a, b = dict_order_csr(ds), dict_order_csr(_Fields(ds))
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    indptr, items, vals = b
    for u, d in ds.i_train_dict.items():
        assert items[indptr[u]:indptr[u + 1]].tolist() == list(d)
        assert vals[indptr[u]:indptr[u + 1]].tolist() == list(d.values())
    assert not all(np.all(np.diff(items[indptr[u]:indptr[u + 1]]) > 0) for u in range(len(ds.users)))   # not sorted


def test_ratings_outside_the_exactness_class_are_refused():
    r = np.random.default_rng(5).integers(1, 6, 600).astype(float)
    SlopeOneModel(_Fields(_dataset(r)), "cuda:0")                       # host only: nothing touches the device yet
    r[7] = 2.3
    with pytest.raises(ValueError, match="SlopeOne"):
        SlopeOneModel(_Fields(_dataset(r)), "cuda:0")
