"""RP3beta without a GPU: the numpy restatement oracle/rp3beta.py against the reference's own goldens (similarity values
and scores bit for bit, W equal but for ties, lists equal at isolated ranks), SciPy's summation order, the model's host
preparation against the oracle, and the C ABI entry points."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import rp3beta as orp3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_G = dict(np.load(os.path.join(ROOT, "tests", "golden", "rp3beta_cases.npz")))
SYMBOLS = ["eb_rp3_tile_cols", "eb_rp3_row_workspace_bytes", "eb_rp3_similarity_f32", "eb_rp3_l1_rows_f32",
           "eb_rp3_prune_workspace_bytes", "eb_rp3_prune_cols_f32", "eb_rp3_score_topk_f32"]


@pytest.mark.parametrize("name", list(_G["cases"]))
def test_oracle_matches_the_reference(name):
    got = orp3.check_case(_G, name)
    assert got["w_nnz"] > 0


def test_goldens_cover_the_issue_grid():
    cases = list(_G["cases"])
    assert {float(_G[f"{c}_alpha"]) for c in cases} == {1.0, 1.0807, 0.5}
    assert {float(_G[f"{c}_beta"]) for c in cases} == {0.6, 0.7029, 0.0}
    assert {bool(_G[f"{c}_normalize"]) for c in cases} == {True, False}
    nb = {int(_G[f"{c}_neighborhood"]) for c in cases}
    assert 10 in nb and -1 in nb and any(k > _G[f"{c}_R"].shape[1] for c in cases for k in [int(_G[f"{c}_neighborhood"])])
    for c in cases:
        R = _G[f"{c}_R"].astype(np.float64)
        assert R.shape[1] <= 300
        assert not R[:, -2].any() and not R[-3].any() and np.array_equal(R[:, 0], R[:, 1])


def _unsorted_csr(g, U, I, dens):
    R = (g.random((U, I)) < dens) * g.integers(1, 11, (U, I)) / 2.0
    r, c = np.nonzero(R)
    perm = np.concatenate([g.permutation(np.flatnonzero(r == u)) for u in range(U)]).astype(np.int64)
    M = sp.csr_matrix((U, I), dtype=np.float32)
    M.indptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=U))]).astype(np.int32)
    M.indices, M.data = c[perm].astype(np.int32), R[r[perm], c[perm]].astype(np.float32)
    return M


def test_scipy_sums_in_the_left_rows_stored_order():
    g = np.random.default_rng(5)
    A = _unsorted_csr(g, 120, 90, 0.2)
    assert not A.has_sorted_indices
    B = sp.random(90, 150, density=0.1, format="csr", dtype=np.float32, random_state=3)
    B.data = (g.random(B.nnz) * 10.0 ** g.integers(-4, 1, B.nnz)).astype(np.float32)
    want = (A @ B).toarray()
    got = orp3.preds(A, B)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_host_preparation_matches_the_oracle():
    from elliot_b200.recommender.rp3beta import RP3Model, l1_rows

    class _Data:
        pass
    g = np.random.default_rng(9)
    d = _Data()
    d.sp_i_train_ratings = _unsorted_csr(g, 150, 70, 0.15)
    d.sp_i_train_ratings.data *= np.float32(1.37)              # values whose fp64 row sums are not exact in fp32
    R = d.sp_i_train_ratings
    assert np.array_equal(l1_rows(R.indptr, R.data).view(np.int32), orp3.l1_rows(R.indptr, R.data).view(np.int32))
    for alpha, beta in [(1.0, 0.6), (1.0807, 0.7029), (0.5, 0.0)]:
        m = RP3Model(d, 10, alpha, beta, False, "cpu")
        (pp, pi, pv), (qp, qi, qv), degree = m.host_operands()
        Pui, Piu, deg = orp3.prepare(R, alpha, beta)
        Ps = Pui.sorted_indices()
        assert np.array_equal(pp, Ps.indptr) and np.array_equal(pi, Ps.indices)
        assert np.array_equal(pv.view(np.int32), Ps.data.view(np.int32))
        assert np.array_equal(qp, Piu.indptr) and np.array_equal(qi, Piu.indices)
        assert np.array_equal(qv.view(np.int32), Piu.data.view(np.int32))
        assert np.array_equal(degree.view(np.int64), deg.view(np.int64))
    assert np.array_equal(R.data, d.sp_i_train_ratings.data), "the DataSet must not change"


def test_model_refuses_bad_parameters():
    from elliot_b200.recommender.rp3beta import RP3Model

    class _Data:
        sp_i_train_ratings = sp.csr_matrix(np.array([[1.0, 0.0], [0.0, -2.0]], np.float32))
    with pytest.raises(ValueError, match="nonnegative"):
        RP3Model(_Data, 10, 1.0, 0.6, False, "cpu")
    _Data.sp_i_train_ratings = abs(_Data.sp_i_train_ratings)
    with pytest.raises(ValueError, match="neighborhood"):
        RP3Model(_Data, 0, 1.0, 0.6, False, "cpu")


def test_header_and_library_declare_the_rp3_entry_points():
    from elliot_b200._lib import SIGNATURES
    from elliot_b200.build import build
    hdr = open(os.path.join(ROOT, "include", "elliot_b200.h")).read()
    lib_path, _ = build()
    L = ctypes.CDLL(lib_path)
    for s in SYMBOLS:
        assert f"{s}(" in hdr and s in SIGNATURES and hasattr(L, s), s
