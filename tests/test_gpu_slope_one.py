"""SlopeOne on the GPU: the deviation kernel against numpy, the ordered fp64 scorer against the oracle (values bit for
bit, lists under the (score desc, item asc) rule), the model against the reference's goldens on every case, reruns, the
restore refusal, and the reference's run_experiment on the SlopeOne block at C1 scale."""
import os

import numpy as np
import pytest
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, dev_csr, to_dev
from elliot_b200 import ops
from oracle import slope_one as oso

pytestmark = pytest.mark.gpu
_G = dict(np.load(os.path.join(GOLD, "slope_one_cases.npz")))
CASES = list(_G["cases"])


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(a, b):
    """Bit-equal fp64 arrays, except that any NaN matches any NaN (the sentinel of E)."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(_bits(np.where(na, 0.0, a)), _bits(np.where(nb, 0.0, b)))


def _case(name):
    return (int(_G[f"{name}_n_items"]), _G[f"{name}_indptr"], _G[f"{name}_items"].astype(np.int64),
            _G[f"{name}_ratings"])


class _Data:
    """The DataSet fields SlopeOneModel reads: i_train_dict in the given dict order."""

    def __init__(self, indptr, items, vals, n_items):
        U = len(indptr) - 1
        self.users, self.items = list(range(U)), list(range(n_items))
        self.i_train_dict = {u: {int(i): float(v) for i, v in zip(items[indptr[u]:indptr[u + 1]], vals[indptr[u]:indptr[u + 1]])}
                             for u in range(U)}


def _train(indptr, items, vals):
    return to_dev(indptr, torch.int64), to_dev(items, torch.int32), to_dev(vals, torch.float32)


def _mask(indptr, items, n_items):
    rows = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    R = np.zeros((len(indptr) - 1, n_items), bool)
    R[rows, items] = True
    return dev_csr(R)[:2]


# ---------------------------------------------------------------- 1. deviations
@pytest.mark.parametrize("n,rows,j0,s", [(1, 1, 0, 0), (37, 16, 8, 1), (2050, 40, 1024, 2), (300, 7, 293, 4)])
def test_dev_kernel_is_bit_equal_to_numpy(n, rows, j0, s):
    g = np.random.default_rng(n)
    F = g.integers(0, 50, (rows, n)).astype(np.float32)
    F[g.random((rows, n)) < 0.3] = 0
    M1 = (g.integers(0, 1 << 20, (rows, n)) * (F > 0)).astype(np.float32)
    M2 = (g.integers(0, 1 << 20, (rows, n)) * (F > 0)).astype(np.float32)
    E = torch.full((j0 + rows + 3, n + 5), 7.0, dtype=torch.float64, device=DEV)
    ops.slope_one_dev_f64(to_dev(F), to_dev(M1), to_dev(M2), n, s, out=E[j0:j0 + rows])
    got = E.cpu().numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        want = np.where(F > 0, (M1.astype(np.float64) - M2) * 2.0 ** -s / F, np.nan)
    assert _same(got[j0:j0 + rows, :n], want), "values or NaN sentinels differ"
    assert np.all(got[:j0] == 7.0) and np.all(got[j0 + rows:] == 7.0) and np.all(got[:, n:] == 7.0)


# ---------------------------------------------------------------- 2. the scorer
def _check_scorer(E, indptr, items, vals, k, users=None):
    """Device top-k against the oracle: every value bit for bit, every list exactly (both use score desc, item asc)."""
    n = E.shape[1]
    mp, mi = _mask(indptr, items, n)
    u_dev = None if users is None else to_dev(users, torch.int32)
    idx, val = ops.slope_one_score_topk(to_dev(E), _train(indptr, items, vals), k, mp, mi, users=u_dev)
    means = oso.user_means(indptr, vals)
    P = oso.scores(E, means, indptr, items, users)
    oi, ov = oso.topk(P, indptr, items, k, users)
    assert np.array_equal(idx.cpu().numpy(), oi)
    assert np.array_equal(_bits(val.cpu().numpy()), _bits(ov))
    return idx, val


@pytest.mark.parametrize("name", CASES)
def test_scorer_matches_the_oracle_on_the_golden_cases(name):
    I, indptr, items, vals = _case(name)
    _, E = oso.deviations(indptr, items, vals, I)
    _check_scorer(E, indptr, items, vals, 37)
    users = np.array([1, 0, 5, len(indptr) - 2, 5])          # fewer than k candidates, one item, a repeat
    _check_scorer(E, indptr, items, vals, 1024, users)


def test_scorer_beyond_one_column_tile_with_cold_items():
    g = np.random.default_rng(7)
    n = 3 * 4096 + 1000                                      # four of the scorer's 4 096-column tiles
    J = g.choice(n, 60, replace=False)                       # the only rows of E the users read
    Es = g.integers(-40, 41, (60, n)) / g.integers(1, 9, (60, n)).astype(np.float64)
    Es[g.random((60, n)) < 0.2] = np.nan
    Es[:, :3] = np.nan                                       # three items nobody co-rated: their score is the mean
    counts = np.array([1, 12, 30, 60, 45])
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    pos = np.concatenate([g.permutation(60)[:c] for c in counts])
    vals = g.integers(1, 6, pos.size).astype(np.float64)
    Ed = torch.full((n, n), float("nan"), dtype=torch.float64, device=DEV)
    Ed[to_dev(J, torch.int64)] = to_dev(Es)
    items = J[pos]
    mp, mi = _mask(indptr, items, n)
    for k in (10, 1024):
        idx, val = ops.slope_one_score_topk(Ed, _train(indptr, items, vals), k, mp, mi)
        means = oso.user_means(indptr, vals)
        P = oso.scores(Es, means, indptr, pos)                # the same sums over the 60 stored rows
        oi, ov = oso.topk(P, indptr, items, k)
        assert np.array_equal(idx.cpu().numpy(), oi), k
        assert np.array_equal(_bits(val.cpu().numpy()), _bits(ov)), k
    assert len(np.unique(oi[oi >= 0] // 4096)) == 4           # the winners come from every tile


def test_scorer_follows_the_given_order():
    name = "half_stars"
    I, indptr, items, vals = _case(name)
    _, E = oso.deviations(indptr, items, vals, I)
    si, sv = oso.sorted_rows(indptr, items, vals)
    _, a = _check_scorer(E, indptr, items, vals, 1024)
    _, b = _check_scorer(E, indptr, si, sv, 1024)
    assert not np.array_equal(_bits(a.cpu().numpy()), _bits(b.cpu().numpy()))


# ---------------------------------------------------------------- 3. the model against the reference's goldens
def _model(indptr, items, vals, I):
    from elliot_b200.recommender.slope_one import SlopeOneModel
    m = SlopeOneModel(_Data(indptr, items, vals, I), DEV)
    m.initialize()
    return m


@pytest.mark.parametrize("name", CASES)
def test_model_matches_the_reference(name):
    I, indptr, items, vals = _case(name)
    m = _model(indptr, items, vals, I)
    _, E = oso.deviations(indptr, items, vals, I)
    assert _same(m.E.cpu().numpy(), E)
    assert oso.crc(oso.reference_dev(m.E.cpu().numpy())) == int(_G[f"{name}_dev_crc"])
    K = int(_G["topk"])
    mp, mi = _mask(indptr, items, I)
    idx, val = m.topk(K, mp, mi)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    ti, tv = _G[f"{name}_topk_idx"], _G[f"{name}_topk_val"]
    assert np.array_equal(idx >= 0, ti >= 0)
    assert np.array_equal(_bits(val), _bits(tv)), "values differ from the reference's at some rank"
    _, ov = oso.topk(oso.scores(E, oso.user_means(indptr, vals), indptr, items), indptr, items, K + 1)
    iso = oso.isolated(ov)[:, :K]
    assert np.array_equal(idx[iso], ti[iso])
    if name == "all_equal":
        assert not iso.any() and np.all(val[idx >= 0] == 4.0)      # ties only: every score is the mean
        assert np.all(np.diff(idx, axis=1)[(idx[:, 1:] >= 0)] > 0)  # ties by item ascending


def test_rerun_is_bit_identical():
    I, indptr, items, vals = _case("stars")
    a, b = _model(indptr, items, vals, I), _model(indptr, items, vals, I)
    assert torch.equal(a.E.view(torch.int64), b.E.view(torch.int64))
    mp, mi = _mask(indptr, items, I)
    (ia, va), (ib, vb) = a.topk(50, mp, mi), b.topk(50, mp, mi)
    assert torch.equal(ia, ib) and torch.equal(va.view(torch.int64), vb.view(torch.int64))


# ---------------------------------------------------------------- 4. run_experiment at C1 scale
c1 = c1h.c1_fixture("slope_one_c1.npz")


def test_restore_is_refused(c1):
    from elliot_b200 import synth_c1
    _, d, tsv = c1
    out = d / "SlopeOne_restore"
    with pytest.raises(NotImplementedError, match="restore"):
        c1h.run(out, synth_c1.experiment_yaml(tsv, str(out), "SlopeOne", "", meta=("restore: True",)))


@pytest.mark.parametrize("ev", ["host", "device"])
def test_run_experiment_matches_the_reference_run(c1, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / f"SlopeOne_{ev}"
    res = c1h.run(out, synth_c1.slope_one_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n"), ev == "device")
    c1h.assert_metrics(res, g["metrics"].tolist(), g["test_metrics"], "SlopeOne", ev)
    if ev == "device":
        c1h.assert_no_rec_files(out)
        return
    files = sorted(os.listdir(out / "recs"))
    assert files == [str(g["rec_file"])] == ["SlopeOne.tsv"], files
    rec = np.loadtxt(out / "recs" / str(g["rec_file"]), delimiter="\t")
    users = np.unique(g["rec_users"])
    mine = rec[np.isin(rec[:, 0].astype(np.int64), users)]
    gu, gi, gs = g["rec_users"], g["rec_items"], g["rec_scores"]
    assert np.array_equal(np.unique(mine[:, 0]).astype(np.int64), users)
    same = total = 0
    for u in users:
        a, b = mine[mine[:, 0] == u], (gu == u)
        assert len(a) == b.sum() == 10
        assert np.array_equal(_bits(a[:, 2]), _bits(gs[b])), u        # the scores as the rec files print them
        iso = oso.isolated(a[None, :, 2])[0]
        iso[-1] = False                                               # the k+1-th value is not in the file
        assert np.array_equal(a[iso, 1].astype(np.int64), gi[b][iso]), u
        same += iso.sum()
        total += 10
    assert same > 0.5 * total, (same, total)
