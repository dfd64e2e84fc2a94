"""EASE^R on the GPU: the blocked fp64 inverse against numpy, the weights kernel bit for bit, the dense scorer bit for bit
against the sparse one, the model against the reference's goldens, and the reference's run_experiment on an EASER block
at C1 scale."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, dev_csr, to_dev
from elliot_b200 import ops
from elliot_b200._lib import EbError
from elliot_b200.recommender import knn
from oracle import ease as oease
from oracle.knn import isolated, topk as oracle_topk

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
RESIDUAL_C = 1.0       # max |A P - I| <= RESIDUAL_C * n * eps * ||A||_inf * ||P||_inf


def _matrix(kind, n, seed):
    g = np.random.default_rng(seed)
    M = g.standard_normal((n, n))
    if kind == "spd":
        return M @ M.T / n + 0.5 * np.eye(n)
    if kind == "sym_indefinite":
        S = (M + M.T) / 2
        return S + np.diag(g.choice([-1.0, 1.0], n) * 0.3 * np.sqrt(n))
    return M


def _gpu_inverse(A, ld=None):
    n = A.shape[0]
    ld = ld or n
    T = torch.full((n, ld), 7.0, dtype=torch.float64, device=DEV)
    T[:, :n] = to_dev(A)
    ops.inverse_f64(T, n)
    out = T.cpu().numpy()
    assert np.all(out[:, n:] == 7.0), "padding columns must stay untouched"
    return out[:, :n]


def _check_residual(A, P):
    n = A.shape[0]
    res = np.abs(A @ P - np.eye(n)).max()
    bound = RESIDUAL_C * n * EPS * np.abs(A).sum(1).max() * np.abs(P).sum(1).max()
    assert res <= bound, (n, res, bound)
    return res


# ---------------------------------------------------------------- 1. the inverse
@pytest.mark.parametrize("kind", ["general", "spd", "sym_indefinite"])
@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 127, 1000, 3706])
def test_inverse_matches_numpy(kind, n):
    A = _matrix(kind, n, n * 7 + len(kind))
    P = _gpu_inverse(A, ld=n + (3 if n % 2 else 0))
    _check_residual(A, P)
    want = np.linalg.inv(A)
    cond = np.linalg.cond(A, np.inf)
    assert np.abs(P - want).max() <= 10 * n * EPS * cond * np.abs(want).max(), kind
    again = _gpu_inverse(A, ld=n + (3 if n % 2 else 0))
    assert np.array_equal(P.view(np.int64), again.view(np.int64)), "reruns must be bit-identical"


def test_inverse_swaps_rows_at_step_zero_and_with_ld_above_n():
    g = np.random.default_rng(3)
    n = 150
    A = g.standard_normal((n, n))
    A[0, 0] = 0.0
    A[97, 0] = 40.0                                 # the pivot of column 0 is row 97
    A[64, 64] = 1e-300                              # column 64 (second panel) needs a swap too
    P = _gpu_inverse(A, ld=n + 17)
    _check_residual(A, P)
    P2 = _gpu_inverse(np.array([[0.0, 2.0], [4.0, 0.0]]))
    assert np.array_equal(P2, np.array([[0.0, 0.25], [0.5, 0.0]]))


def test_inverse_ties_and_exact_small_cases():
    A = np.array([[1.0, 2.0], [-1.0, 3.0]])        # |a| ties in column 0: the lowest row (0) pivots
    P = _gpu_inverse(A)
    assert np.abs(P - np.linalg.inv(A)).max() <= 4 * EPS
    assert np.array_equal(_gpu_inverse(np.array([[4.0]])), np.array([[0.25]]))


@pytest.mark.parametrize("bad", ["zero_column", "zero_matrix", "nan"])
def test_singular_or_non_finite_matrix_names_the_column(bad):
    g = np.random.default_rng(11)
    n = 150
    A = g.standard_normal((n, n))
    col = {"zero_column": 70, "zero_matrix": 0, "nan": 0}[bad]
    if bad == "zero_column":
        A[:, 70] = 0.0
    elif bad == "zero_matrix":
        A[:] = 0.0
    else:
        A[5, 0] = np.nan
    with pytest.raises(EbError, match=f"column {col}:"):
        _gpu_inverse(A)
    P = _gpu_inverse(_matrix("general", 40, 1))          # the status word is reset by the next call
    _check_residual(_matrix("general", 40, 1), P)


def test_inverse_rejects_bad_arguments():
    A = torch.zeros((4, 4), dtype=torch.float64, device=DEV)
    with pytest.raises(EbError, match="bad shape"):
        ops._call("eb_inverse_f64", A, A.data_ptr(), 4, 3, A.data_ptr(), 1 << 20)
    with pytest.raises(EbError, match="workspace"):
        ops._call("eb_inverse_f64", A, A.data_ptr(), 4, 4, A.data_ptr(), 16)


# ---------------------------------------------------------------- 2. normal matrix and weights
def test_normal_matrix_rows_from_slabs():
    g = np.random.default_rng(2)
    n, S, row0 = 77, 16, 40
    slab = (g.integers(-300, 300, (S, n + 5)) * 4).astype(np.float32)
    count = g.integers(0, 50, n).astype(np.int32)
    A = torch.full((n, n + 2), 9.0, dtype=torch.float64, device=DEV)
    ops.ease_normal_f64(to_dev(slab)[:, :n + 5], row0, to_dev(count), 0.3, 0.25, A)
    got = A.cpu().numpy()
    want = slab[:, :n].astype(np.float64) * 0.25
    for r in range(S):
        want[r, row0 + r] = float(np.float32(count[row0 + r] + 0.3))
    assert np.array_equal(got[row0:row0 + S, :n], want)
    assert np.all(got[:row0] == 9.0) and np.all(got[row0 + S:] == 9.0) and np.all(got[:, n:] == 9.0)


def test_weights_bit_equal_to_numpy():
    g = np.random.default_rng(4)
    n = 333
    P = g.standard_normal((n, n)) * 10.0 ** g.integers(-3, 3, (n, n))
    B = ops.ease_weights_f32(to_dev(P)).cpu().numpy()
    want = (-P / np.diag(P)[None, :]).astype(np.float32)
    want[np.diag_indices(n)] = 0.0
    assert np.array_equal(B.view(np.int32), want.view(np.int32))
    P[40, 40] = 0.0
    P[7, 7] = 0.0
    with pytest.raises(EbError, match="column 7:"):
        ops.ease_weights_f32(to_dev(P))


# ---------------------------------------------------------------- 3. dense scorer
def _score_case(n_rows, n_mid, n_cols, seed):
    g = np.random.default_rng(seed)
    A = sp.random(n_rows, n_mid, density=0.08, random_state=seed, format="csr")
    A.data = g.integers(1, 11, A.nnz) / 2.0
    A = A.tolil(); A[3, :] = 0; A = A.tocsr(); A.eliminate_zeros()          # a row without entries
    B = (g.standard_normal((n_mid, n_cols)) * 1e-2).astype(np.float32)
    B[g.random((n_mid, n_cols)) < 0.1] = 0.0
    if n_cols > 1:
        B[:, 1] = B[:, 0]                                                    # duplicated column: exact ties
    mask = sp.random(n_rows, n_cols, density=0.1, random_state=seed + 2, format="lil")
    if n_cols > 3:
        mask[5, :] = 1; mask[5, n_cols - 1] = 0; mask[5, 1] = 0              # only two unmasked columns
    mask = sp.csr_matrix(mask); mask.data[:] = 1
    return A, B, mask


@pytest.mark.parametrize("n_cols", [1, 300, "tile+77"])
@pytest.mark.parametrize("k", [1, 10, 1024])
@pytest.mark.parametrize("select", ["all", "users", "begin"])
def test_dense_scorer_bit_equal_to_sparse(n_cols, k, select):
    T = ops.knn_score_tile_cols()
    n_cols = T + 77 if n_cols == "tile+77" else n_cols
    A, B, mask = _score_case(96, 70, n_cols, 13 + k)
    dA, dM = dev_csr(A), dev_csr(mask)
    Bcsr = sp.csr_matrix(B)
    Bcsr.sort_indices()
    dBs = dev_csr(Bcsr)
    ldb = n_cols + 5
    dB = torch.zeros((70, ldb), dtype=torch.float32, device=DEV)
    dB[:, :n_cols] = to_dev(B)
    f = knn.frac_bits(knn._bound(dA, dBs))
    kw = {}
    rows = np.arange(96)
    if select == "users":
        rows = np.array([95, 3, 5, 40, 40, 0], np.int32)
        kw = {"users": to_dev(rows)}
    elif select == "begin":
        rows = np.arange(17, 96)
        kw = {"user_begin": 17, "n_sel": len(rows)}
    di, dv = ops.dense_score_topk(dA, dB[:, :n_cols], k, f, dM[0], dM[1], **kw)
    si, sv = ops.knn_score_topk(dA, dBs, n_cols, k, f, dM[0], dM[1], **kw)
    assert torch.equal(di, si)
    assert torch.equal(dv.view(torch.int32), sv.view(torch.int32))
    # against an fp64 numpy top-k: values within the fixed-point bound, the same column at every isolated rank
    P = (A @ B.astype(np.float64))[rows]
    M = mask.toarray()[rows] != 0
    oi, ov = oracle_topk(P, M, k)
    gi, gv = di.cpu().numpy(), dv.cpu().numpy().astype(np.float64)
    filled = oi >= 0
    assert np.array_equal(gi >= 0, filled)
    nterms = np.diff(A.indptr)[rows]
    with np.errstate(invalid="ignore"):
        tol = np.spacing(np.abs(ov).astype(np.float32)).astype(np.float64) + nterms[:, None] * 2.0 ** -(f + 1)
    assert np.all(np.abs(gv[filled] - ov[filled]) <= tol[filled])
    iso = filled.copy()
    with np.errstate(invalid="ignore"):
        iso[:, 1:] &= (ov[:, :-1] - ov[:, 1:]) > 2 * tol[:, 1:]
        iso[:, :-1] &= (ov[:, :-1] - ov[:, 1:]) > 2 * tol[:, :-1]
    assert np.array_equal(gi[iso], oi[iso])


# ---------------------------------------------------------------- 4. the model against the reference's goldens
class _Data:
    def __init__(self, R):
        self.sp_i_train_ratings = sp.csr_matrix(R.astype(np.float32))


_G = dict(np.load(os.path.join(GOLD, "ease_cases.npz")))


@pytest.mark.parametrize("name", list(_G["cases"]))
def test_model_matches_reference_goldens(name):
    from elliot_b200.recommender.ease import EASEModel
    g = _G
    R = g[f"{name}_R"].astype(np.float64)
    lam, k = float(g[f"{name}_l2_norm"]), int(g["topk"])
    data = _Data(R)
    before = [a.tobytes() for a in (data.sp_i_train_ratings.data, data.sp_i_train_ratings.indices,
                                    data.sp_i_train_ratings.indptr)]
    m = EASEModel(data, lam, DEV)
    m.initialize()
    B_or = oease.weights(np.linalg.inv(oease.normal_matrix(R, lam)))
    # both round an fp64 quotient to fp32 once; the two fp64 inverses differ in the last bits only, so at most 1 ulp apart
    assert np.all(np.abs(m.B.cpu().numpy() - B_or) <= np.spacing(np.abs(B_or))), name
    mask = dev_csr(R != 0)
    ti, tv = m.topk(k, mask[0], mask[1])
    gi, gv = ti.cpu().numpy(), tv.cpu().numpy().astype(np.float64)
    ri, rv = g[f"{name}_topk_idx"], g[f"{name}_topk_val"]
    _, ov = oracle_topk(oease.preds(R, B_or), R != 0, k + 1)
    iso = isolated(ov[:, :k], ov[:, k])
    assert np.array_equal(gi[iso], ri[iso]), name
    ok = np.isfinite(rv)
    assert np.array_equal(gi >= 0, ok), name
    scale = np.abs(g[f"{name}_preds"]).max()
    assert np.abs(gv[ok] - rv[ok]).max() <= 1e-5 * scale, name
    after = [a.tobytes() for a in (data.sp_i_train_ratings.data, data.sp_i_train_ratings.indices,
                                   data.sp_i_train_ratings.indptr)]
    assert before == after, "the DataSet must not change"


def test_model_rerun_is_bit_identical():
    from elliot_b200.recommender.ease import EASEModel
    R = _G["int_l1000_R"].astype(np.float64)
    Bs = []
    for _ in range(2):
        m = EASEModel(_Data(R), 1e3, DEV)
        m.initialize()
        Bs.append(m.B.cpu().numpy())
    assert np.array_equal(Bs[0].view(np.int32), Bs[1].view(np.int32))


def test_singular_normal_matrix_names_l2_norm():
    from elliot_b200.recommender.ease import EASEModel
    R = _G["int_l0.3_tiny_R"].astype(np.float64)          # a cold item: with l2_norm 0 its row and column are zero
    m = EASEModel(_Data(R), 0.0, DEV)
    with pytest.raises(ValueError, match="l2_norm"):
        m.initialize()


def test_ratings_without_an_exact_scale_are_refused():
    from elliot_b200.recommender.ease import EASEModel
    R = np.array([[1.0, 0.3], [0.0, 2.0]])
    with pytest.raises(ValueError, match="EASER needs ratings"):
        EASEModel(_Data(R), 1e3, DEV).initialize()


# ---------------------------------------------------------------- 5. run_experiment at C1 scale
c1 = c1h.c1_fixture("ease_c1.npz")


@pytest.mark.parametrize("ev", ["host", "device"])
def test_run_experiment_matches_the_reference_run(c1, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / ev
    res = c1h.run(out, synth_c1.ease_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n"), ev == "device")
    c1h.assert_metrics(res, g["metrics"].tolist(), g["test_metrics"], ev)
    if ev == "device":
        c1h.assert_no_rec_files(out)
        return
    files = os.listdir(out / "recs")
    assert files == [str(g["rec_file"])], (files, str(g["rec_file"]))          # the same model `name` as the reference's
    rec = np.loadtxt(out / "recs" / files[0], delimiter="\t")
    mine = rec[np.isin(rec[:, 0].astype(np.int64), np.unique(g["rec_users"]))]
    assert np.array_equal(mine[:, 0].astype(np.int64), g["rec_users"])
    assert np.array_equal(mine[:, 1].astype(np.int64), g["rec_items"])
    assert np.allclose(mine[:, 2], g["rec_scores"], rtol=1e-4, atol=1e-5 * np.abs(g["rec_scores"]).max())
