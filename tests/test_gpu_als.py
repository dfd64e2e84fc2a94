"""iALS / WRMF on the GPU: the fp64 Gram and the batched normal-equation solve against numpy, both models against the
reference's goldens after every epoch, and the reference's run_experiment on iALS and WRMF blocks at C1 scale."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, to_dev
from elliot_b200 import ops
from elliot_b200._lib import EbError

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- 1. Gram
@pytest.mark.parametrize("d", [1, 8, 10, 33, 64, 200])
@pytest.mark.parametrize("n", [1, 255, 1000, 40_003])
def test_gram_matches_numpy_and_reruns_bit_identical(n, d):
    g = np.random.default_rng(n * 1000 + d)
    ld = d + 3
    Y = g.standard_normal((n, ld))
    Yd = to_dev(Y)
    G1 = ops.gram_f64(Yd, d).cpu().numpy()
    G2 = ops.gram_f64(Yd.clone(), d).cpu().numpy()
    want = Y[:, :d].T @ Y[:, :d]
    assert np.array_equal(G1, G2)
    assert np.array_equal(G1, G1.T)
    assert np.abs(G1 - want).max() <= 1e-13 * np.abs(want).max()


def test_gram_rejects_bad_arguments():
    Y = torch.zeros((4, 201), dtype=torch.float64, device=DEV)
    with pytest.raises(EbError, match="outside"):
        ops.gram_f64(Y, 201)
    with pytest.raises(EbError, match="workspace"):
        ops._call("eb_gram_f64", Y, Y.data_ptr(), 4, 8, 201, Y.data_ptr(), 0, 0)


# ---------------------------------------------------------------- 2. Solve
def _system(n_rows, n_cols, d, lens, seed, w_kind="random"):
    """Random rows with the given entry counts over a random table Y; w, c arbitrary (w may be negative, A stays
    positive definite through G and reg)."""
    g = np.random.default_rng(seed)
    Y = g.standard_normal((n_cols, d)) * 0.3
    indptr = np.zeros(n_rows + 1, np.int64)
    indptr[1:] = np.cumsum(lens)
    nnz = int(indptr[-1])
    indices = np.concatenate([np.sort(g.choice(n_cols, size=l, replace=l > n_cols)) for l in lens]).astype(np.int32) \
        if nnz else np.zeros(0, np.int32)
    w = g.uniform(-0.05, 3.0, nnz) if w_kind == "random" else np.full(nnz, 1.5)
    c = g.uniform(0.0, 4.0, nnz)
    G = Y.T @ Y
    return Y, G, indptr, indices, w, c


def _numpy_solve(Y, G, indptr, indices, w, c, reg):
    d = Y.shape[1]
    X = np.empty((len(indptr) - 1, d))
    for r in range(len(indptr) - 1):
        s = slice(indptr[r], indptr[r + 1])
        P = Y[indices[s]]
        A = G + (P * w[s][:, None]).T @ P + reg * np.eye(d)
        X[r] = np.linalg.solve(A, P.T @ c[s])
    return X


def _gpu_solve(Y, G, indptr, indices, w, c, reg, order, ld_x=None):
    d = Y.shape[1]
    ld_x = ld_x or d
    X = torch.full((len(indptr) - 1, ld_x), 7.0, dtype=torch.float64, device=DEV)
    ops.als_solve_f64(to_dev(G), to_dev(Y), d, to_dev(indptr), to_dev(indices), to_dev(w), to_dev(c), to_dev(order.astype(np.int32)), reg, X)
    return X.cpu().numpy()


@pytest.mark.parametrize("d", [1, 10, 32, 33, 64, 200])
def test_solve_matches_numpy_both_mappings(d):
    lens = [0, 1, 2, 17, 5_003, 40, 0, 3, 250, 1]
    Y, G, indptr, indices, w, c = _system(len(lens), 6000, d, lens, seed=d)
    reg = 0.1
    want = _numpy_solve(Y, G, indptr, indices, w, c, reg)
    order = np.argsort(-np.diff(indptr), kind="stable")
    got = _gpu_solve(Y, G, indptr, indices, w, c, reg, order, ld_x=d + 2)
    assert np.all(got[:, d:] == 7.0), "padding columns must stay untouched"
    got = got[:, :d]
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < 1e-11, err
    assert np.all(got[[0, 6]] == 0.0), "rows without entries solve to 0"
    perm = np.random.default_rng(1).permutation(len(lens))
    again = _gpu_solve(Y, G, indptr, indices, w, c, reg, perm, ld_x=d + 2)[:, :d]
    assert np.array_equal(got, again), "the result must not depend on the row order"


@pytest.mark.parametrize("d", [10, 64])
def test_solve_many_rows_and_partial_order(d):
    g = np.random.default_rng(5)
    lens = g.integers(0, 60, 3000)
    Y, G, indptr, indices, w, c = _system(len(lens), 500, d, lens, seed=7)
    want = _numpy_solve(Y, G, indptr, indices, w, c, 0.05)
    order = np.argsort(-np.diff(indptr), kind="stable")
    keep = order[order % 3 != 0]                       # rows left out of `order` are not written
    got = _gpu_solve(Y, G, indptr, indices, w, c, 0.05, keep)
    out = np.arange(len(lens)) % 3 == 0
    assert np.all(got[out] == 7.0)
    err = np.abs(got[~out] - want[~out]).max() / np.abs(want).max()
    assert err < 1e-11, err
    again = _gpu_solve(Y, G, indptr, indices, w, c, 0.05, g.permutation(keep))
    assert np.array_equal(got, again)


@pytest.mark.parametrize("d", [10, 48])
def test_solve_reports_the_first_indefinite_row(d):
    lens = [3, 4, 5, 6, 7]
    Y, G, indptr, indices, w, c = _system(len(lens), 50, d, lens, seed=3, w_kind="fixed")
    w = w.copy()
    for r in (3, 1):                                   # rows 1 and 3 get a strongly negative weight
        w[indptr[r]] = -1e6
    order = np.arange(len(lens))[::-1].copy()
    with pytest.raises(EbError, match="row 1:"):
        _gpu_solve(Y, G, indptr, indices, w, c, 0.1, order)
    with pytest.raises(EbError, match="row 0:"):       # reg <= 0 with G = 0 and a row without entries
        _gpu_solve(Y, np.zeros((d, d)), np.array([0, 0], np.int64), np.zeros(0, np.int32), np.zeros(0), np.zeros(0), 0.0,
                   np.array([0]))


def test_solve_rejects_bad_arguments():
    G = torch.zeros((201, 201), dtype=torch.float64, device=DEV)
    e = torch.zeros(1, dtype=torch.int64, device=DEV)
    i = torch.zeros(1, dtype=torch.int32, device=DEV)
    v = torch.zeros(1, dtype=torch.float64, device=DEV)
    with pytest.raises(EbError, match="outside"):
        ops.als_solve_f64(G, G, 201, e, i, v, v, i, 0.1, G)
    with pytest.raises(EbError, match="bad shape"):
        ops._call("eb_als_solve_f64", G, G.data_ptr(), G.data_ptr(), 5, 10, e.data_ptr(), i.data_ptr(), v.data_ptr(),
                  v.data_ptr(), i.data_ptr(), 1, 0.1, G.data_ptr(), 10)
    with pytest.raises(EbError, match="misaligned"):
        ops._call("eb_als_solve_f64", G, G.data_ptr() + 4, G.data_ptr(), 10, 10, e.data_ptr(), i.data_ptr(), v.data_ptr(),
                  v.data_ptr(), i.data_ptr(), 1, 0.1, G.data_ptr(), 10)


# ---------------------------------------------------------------- 3. Both models against the reference's goldens
class _Data:
    """The DataSet fields ALSModel reads; public ids == private ids."""

    def __init__(self, R):
        rows, cols = np.nonzero(R)
        self.sp_i_train = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), dtype=np.float32, shape=R.shape)
        self.users, self.items = list(range(R.shape[0])), list(range(R.shape[1]))


def _case(g, name):
    d, alpha, eps, reg = g[f"{name}_hp"].tolist()
    kind = "iALS" if name.startswith("ials") else "WRMF"
    if kind == "WRMF" and float(alpha).is_integer():
        alpha = int(alpha)
    return kind, int(d), alpha, (1.0 if np.isnan(eps) else eps), reg, str(g[f"{name}_scaling"])


_G = dict(np.load(os.path.join(GOLD, "als_cases.npz")))
GOLDEN_TOL = 1e-9          # max abs difference over max abs value, every epoch


@pytest.mark.parametrize("name", list(_G["cases"]))
def test_model_matches_reference_every_epoch(name):
    from elliot_b200.recommender.als import ALSModel
    g = _G
    kind, d, alpha, eps, reg, scaling = _case(g, name)
    R = g[f"{name}_R"].astype(np.float64)
    data = _Data(R)
    before = [a.tobytes() for a in (data.sp_i_train.data, data.sp_i_train.indices, data.sp_i_train.indptr)]
    np.random.seed(42)                                   # what init_charger does before the model is built
    m = ALSModel(kind, d, data, alpha, reg, eps, scaling if kind == "iALS" else "linear", DEV)
    assert np.array_equal(m.X.cpu().numpy(), g[f"{name}_X0"]) and np.array_equal(m.Y.cpu().numpy(), g[f"{name}_Y0"])
    worst = 0.0
    for e in range(int(g["epochs"])):
        m.train_step()
        for got, want in ((m.X, g[f"{name}_X"][e]), (m.Y, g[f"{name}_Y"][e])):
            err = np.abs(got.cpu().numpy() - want).max() / np.abs(want).max()
            worst = max(worst, err)
            assert err <= GOLDEN_TOL, (name, e, err)
    print(f"\n{name}: tables within {worst:.2e} (max abs diff / max abs value) of the reference over every epoch")
    mask = sp.csr_matrix(R != 0)
    mask.sort_indices()
    idx, val = m.topk(int(g["topk"]), to_dev(mask.indptr, torch.int64), to_dev(mask.indices, torch.int32))
    assert np.array_equal(idx.cpu().numpy(), g[f"{name}_topk_idx"]), name
    tv = g[f"{name}_topk_val"]
    assert np.abs(val.cpu().numpy() - tv).max() <= GOLDEN_TOL * np.abs(tv).max()
    after = [a.tobytes() for a in (data.sp_i_train.data, data.sp_i_train.indices, data.sp_i_train.indptr)]
    assert before == after, "the DataSet's sp_i_train must not change (the reference's iALS rewrites it)"


def test_rerun_is_bit_identical():
    from elliot_b200.recommender.als import ALSModel
    R = _G["ials_log_d33_R"].astype(np.float64)
    tables = []
    for _ in range(2):
        np.random.seed(3)
        m = ALSModel("iALS", 33, _Data(R), 2.5, 0.5, 0.3, "log", DEV)
        m.train_step(); m.train_step()
        tables.append((m.X.cpu().numpy(), m.Y.cpu().numpy()))
    assert all(np.array_equal(a, b) for a, b in zip(*tables))


def test_negative_alpha_is_refused_with_its_name():
    from elliot_b200.recommender.als import ALSModel
    R = _G["wrmf_d10_R"].astype(np.float64)
    np.random.seed(0)
    m = ALSModel("iALS", 10, _Data(R), -50.0, 0.1, 1.0, "linear", DEV)
    with pytest.raises(ValueError, match="alpha"):
        m.train_step()


# ---------------------------------------------------------------- 4. run_experiment at C1 scale
c1 = c1h.c1_fixture("als_c1.npz")


BLOCKS = {
    "iALS": "      factors: 10\n      alpha: 1\n      epsilon: 1\n      reg: 0.1\n      scaling: linear\n",
    "WRMF": "      factors: 10\n      alpha: 1\n      reg: 0.1\n",
}


@pytest.mark.parametrize("ev", ["host", "device"])
@pytest.mark.parametrize("model", ["iALS", "WRMF"])
def test_run_experiment_matches_the_reference_run(c1, model, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    p = model.lower()
    epochs = int(g[f"{p}_epochs"])
    out = d / f"{model}_{ev}"
    res = c1h.run(out, synth_c1.als_yaml(tsv, str(out), model, epochs, BLOCKS[model], model_extra=f"      b200_eval: {ev}\n"),
                  ev == "device")
    assert len(res["history"]) == epochs
    c1h.assert_metrics(res, g["metrics"].tolist(), g[f"{p}_test_metrics"], model, ev)
    if ev == "device":
        c1h.assert_no_rec_files(out)
        return
    files = sorted(os.listdir(out / "recs"))
    assert files == g[f"{p}_rec_files"].tolist(), (files, g[f"{p}_rec_files"])      # same model `name` as the reference's
    rec = np.loadtxt(out / "recs" / str(g[f"{p}_rec_file"]), delimiter="\t")     # the last epoch's lists
    users = np.unique(g[f"{p}_rec_users"])
    mine = rec[np.isin(rec[:, 0].astype(np.int64), users)]
    assert np.array_equal(mine[:, 0].astype(np.int64), g[f"{p}_rec_users"])
    assert np.array_equal(mine[:, 1].astype(np.int64), g[f"{p}_rec_items"])
    assert np.allclose(mine[:, 2], g[f"{p}_rec_scores"], rtol=1e-6, atol=1e-9)
