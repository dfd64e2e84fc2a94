"""CPU tests of MostPop and Random: oracle/unpersonalized.py against the dicts the reference's own classes returned
(tests/golden/unpersonalized_cases.npz, minted by oracle/gen_golden_unpersonalized.py), including the private-key quirk,
int scores, n_u of 0 and 1, rejection extremes and a second call that continues the stream; and the host evaluator
against the reference Evaluator's metrics on those lists, whose Random lists hold the same item more than once."""
from types import SimpleNamespace

import numpy as np
import pytest

import unpersonalized_cases as uc
from elliot_b200.evaluation import Evaluator
from oracle import unpersonalized as oun


def mostpop_dict(data, rows, pop, skipped):
    r = {}
    for u in range(data.num_users):
        if skipped[u]:
            r[u] = []
        else:
            r[data.users[u]] = [(data.items[i], int(p)) for i, p in zip(rows[u], pop[u]) if i >= 0]
    return r


def test_mostpop_oracle_equals_reference():
    g = uc.case("mostpop")
    data = uc.data_of(g)
    indptr, indices = uc.train_csr(data)
    rows, pop, skipped = oun.mostpop(indptr, indices, data.num_items, int(g["k"]))
    want = uc.golden_dict(g)
    assert uc.same_dict(mostpop_dict(data, rows, pop, skipped), want)
    assert skipped.sum() == 2
    # key 5 is private user 5's empty list, overwritten by the user whose public id is 5; key 20 is the reverse
    assert want[5] != [] and want[20] == []
    assert data.users[5] not in want and data.users[20] not in want
    # pop ties are listed by private item ascending
    p = oun.popularity(indptr, indices, data.num_items)[0]
    assert len(np.unique(p)) < data.num_items


@pytest.mark.parametrize("name", uc.RANDOM)
def test_random_oracle_equals_reference_over_two_calls(name):
    g = uc.case(name)
    data = uc.data_of(g)
    indptr, indices = uc.train_csr(data)
    stream = oun.Stream(int(g["seed"]))
    for call in range(2):
        r = oun.random_draws(stream, indptr, data.num_items, int(g["k"]))
        idx = oun.complement_select(r, indptr, indices, data.num_items)
        got = {data.users[u]: [(data.items[i], 1) for i in idx[u] if i >= 0] for u in range(data.num_users)}
        assert uc.same_dict(got, uc.golden_dict(g, call)), call
        assert stream.consumed == int(g[f"consumed_{call}"]), call
    n_u = data.num_items - np.diff(indptr)
    assert {0, 1, 3, 32, 33} <= set(n_u.tolist())


def test_stream_reads_like_numpy_randint():
    s, rs = oun.Stream(3, chunk=7), np.random.RandomState(3)
    for n in (1, 2, 5, 32, 33, 1000, 1, 2 ** 20 + 1):
        assert s.randint(n) == rs.randint(n)


@pytest.mark.parametrize("name", uc.CASES)
def test_host_evaluator_equals_reference(name):
    g = uc.case(name)
    data = uc.data_of(g)
    names = g["metrics"].tolist()
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    for call in range(2 if f"keys_1" in g else 1):
        recs = uc.golden_dict(g, call)
        res = ev.eval((recs, recs))
        for c, k in enumerate(uc.CUTOFFS):
            for m, w in zip(names, g[f"values_{call}"][c].tolist()):
                got = res[k]["test_results"][m]
                assert abs(got - w) <= 1e-12 * max(1.0, abs(w)), (name, call, k, m, got, w)
