"""PureSVD on the GPU: the sparse products, the pivoted CholeskyQR, the tall-times-small product and the Jacobi
eigensolver against numpy; the model against the fp64 oracle and the reference's goldens on every case; reruns; the
factor limit; and the reference's run_experiment on the docstring's PureSVD block at C1 scale."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, dev_csr, to_dev
from elliot_b200 import ops
from oracle import pure_svd as opsvd
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
_G = dict(np.load(os.path.join(GOLD, "pure_svd_cases.npz")))
ORACLE_TOL = 1e-9           # scores: max |dP| / max |P| against the fp64 oracle


class _Data:
    def __init__(self, R):
        self.sp_i_train = sp.csr_matrix(R.astype(np.float32))


def _fit(R, factors, seed=42):
    from elliot_b200.recommender.pure_svd import PureSVDModel
    m = PureSVDModel(factors, _Data(R), seed, DEV)
    m.train_step()
    return m


def _host(m):
    return m.user_vec.cpu().numpy(), m.item_vec.cpu().numpy(), m.s.cpu().numpy()


# ---------------------------------------------------------------- 1. the pieces
@pytest.mark.parametrize("w", [1, 20, 45, 100, 200])
def test_spmm_matches_scipy_and_reruns_bit_identical(w):
    g = np.random.default_rng(w)
    A = sp.random(700, 300, density=0.05, random_state=w, dtype=np.float32, format="csr")
    A.data[:] = g.integers(1, 6, A.nnz)
    A[5] = 0                                                  # a row without entries
    A.eliminate_zeros()
    X = g.standard_normal((300, w))
    Ad = dev_csr(A)
    Y1 = ops.csr_spmm_f64(Ad, to_dev(X)).cpu().numpy()
    Y2 = ops.csr_spmm_f64(Ad, to_dev(X)).cpu().numpy()
    want = A.astype(np.float64) @ X
    assert np.array_equal(Y1, Y2)
    assert np.all(Y1[5] == 0.0)
    assert np.abs(Y1 - want).max() <= 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("n,w,rank", [(500, 20, 20), (500, 45, 17), (60, 45, 39), (3000, 200, 200), (150, 200, 150)])
def test_cholesky_qr_matches_the_oracle(n, w, rank):
    g = np.random.default_rng(n + w)
    X = g.standard_normal((n, rank)) @ g.standard_normal((rank, w))
    X[:, 3] = X[:, 1]
    Xd = to_dev(X)
    G = ops.gram_f64(Xd, w)
    r = torch.zeros(1, dtype=torch.int32, device=DEV)
    M = ops.chol_pivoted_f64(G, rank=r).cpu().numpy()
    Mo, ro = opsvd.chol_pivoted(G.cpu().numpy())
    want_rank = min(rank, w - 1)
    assert int(r.item()) == ro == want_rank
    assert np.abs(M - Mo).max() <= 1e-9 * np.abs(Mo).max()
    Y = ops.tall_times_small_f64(Xd, to_dev(M))
    assert np.abs(Y.cpu().numpy() - X @ M).max() <= 1e-12 * np.abs(X @ M).max()
    ops.tall_times_small_f64(Xd, to_dev(M), out=Xd)           # in place
    assert torch.equal(Xd, Y)
    ops.tall_times_small_f64(Xd, ops.chol_pivoted_f64(ops.gram_f64(Xd, w)), out=Xd)    # the second pass
    Yn = Xd.cpu().numpy()
    assert np.all(Yn[:, want_rank:] == 0.0)
    assert np.abs(Yn[:, :want_rank].T @ Yn[:, :want_rank] - np.eye(want_rank)).max() < 1e-12


def test_row_strided_out_matches_contiguous_out():
    """The sparse and tall-times-small products write row blocks with unit column stride: a [:, :w] view of a wider
    buffer receives the same bits as a contiguous output, and its padding columns are left alone."""
    g = np.random.default_rng(3)
    A = sp.random(500, 300, density=0.05, random_state=3, dtype=np.float32, format="csr")
    A.data[:] = g.integers(1, 6, A.nnz)
    Ad, X, M = dev_csr(A), to_dev(g.standard_normal((300, 20))), to_dev(g.standard_normal((20, 12)))
    wide = torch.full((500, 32), float("nan"), dtype=torch.float64, device=DEV)
    Y = ops.csr_spmm_f64(Ad, X)
    assert torch.equal(ops.csr_spmm_f64(Ad, X, out=wide[:, :20]), Y) and torch.isnan(wide[:, 20:]).all()
    wide = torch.full((500, 16), float("nan"), dtype=torch.float64, device=DEV)
    Z = ops.tall_times_small_f64(Y, M)
    assert torch.equal(ops.tall_times_small_f64(Y, M, out=wide[:, :12]), Z) and torch.isnan(wide[:, 12:]).all()


@pytest.mark.parametrize("w,rank", [(1, 1), (2, 2), (20, 20), (45, 30), (199, 199), (200, 120)])
def test_jacobi_eigensolver_matches_eigh(w, rank):
    g = np.random.default_rng(w)
    B = g.standard_normal((rank, w)) * np.linspace(3, 0.1, rank)[:, None]
    A = B.T @ B
    lam, V = ops.sym_eig_f64(to_dev(A))
    lam, V = lam.cpu().numpy(), V.cpu().numpy()
    want = np.linalg.eigvalsh(A)[::-1]
    off = 4 * w * 2.0 ** -52 * np.trace(A)        # the rotations stop at off-diagonal entries of w eps trace(A)
    assert np.all(np.diff(lam) <= 0)
    assert np.abs(lam - want).max() <= off
    assert np.abs(V.T @ V - np.eye(w)).max() < 1e-12
    assert np.abs(A @ V - V * lam).max() <= w * off
    lam2, V2 = ops.sym_eig_f64(to_dev(A))
    assert np.array_equal(lam2.cpu().numpy(), lam) and np.array_equal(V2.cpu().numpy(), V)


# ---------------------------------------------------------------- 2. the model against the oracle and the goldens
@pytest.mark.parametrize("name", list(_G["cases"]))
def test_model_matches_oracle_and_reference(name):
    R = _G[f"{name}_R"].astype(np.float64)
    f = int(_G[f"{name}_factors"])
    m = _fit(R, f, int(_G["seed"]))
    user, item, s = _host(m)
    assert np.all(np.isfinite(user)) and np.all(np.isfinite(item)) and np.all(np.isfinite(s))
    ou, oi, os_ = opsvd.fit(R, f, int(_G["seed"]))
    assert user.shape == ou.shape and item.shape == oi.shape
    assert np.abs(s - os_).max() <= 1e-12 * os_[0]
    P, Po = user @ item.T, ou @ oi.T
    err = np.abs(P - Po).max() / np.abs(Po).max()
    assert err <= ORACLE_TOL, err
    cc = opsvd.clear_columns(os_, ou)
    for a, b in ((user, ou), (item, oi)):
        assert np.abs(a[:, cc] - b[:, cc]).max() <= 1e-7 * np.abs(b).max(), name
    print(f"\n{name}: scores within {err:.1e} max|P| of the oracle, {cc.sum()} determined columns")
    # the reference: s, scores, orientation, lists at isolated ranks (fp32 level)
    case = {"R": R, "s": _G[f"{name}_s"], "user_vec": _G[f"{name}_user_vec"], "item_vec": _G[f"{name}_item_vec"],
            "topk_idx": _G[f"{name}_topk_idx"]}
    opsvd.check_against(case, user, item, s)
    # the device's top-k: exact against its own fp64 tables (unit 2^-53), the reference's at isolated ranks
    K = int(_G["topk"])
    mask = dev_csr(R != 0)
    idx, val = m.topk(K, mask[0], mask[1])
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    mp, mi = mask[0].cpu().numpy(), mask[1].cpu().numpy()
    q, n = check_topk_fp64(user, item, None, m.d, K, mp, mi, np.arange(R.shape[0]), idx, val, 2.0 ** -53)
    assert n > 0
    Pm = np.where(R != 0, -np.inf, P)
    ov = -np.sort(-Pm, axis=1)[:, :K + 1]
    iso = opsvd.isolated_abs(ov[:, :K], ov[:, K], 1e-5 * np.abs(P).max())
    assert np.array_equal(idx[iso], case["topk_idx"][iso]), name


def test_rerun_is_bit_identical():
    for name in ("wide_f10_it7", "tall_f190"):
        R = _G[f"{name}_R"].astype(np.float64)
        f = int(_G[f"{name}_factors"])
        a, b = _host(_fit(R, f)), _host(_fit(R, f))
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), name


def test_factors_past_the_block_width_are_refused():
    R = _G["tall_f10_it4_R"].astype(np.float64)
    with pytest.raises(ValueError, match="factors"):
        _fit(R, 191)
    with pytest.raises(ValueError, match="factors"):
        _fit(R, 0)


# ---------------------------------------------------------------- 3. run_experiment at C1 scale
c1 = c1h.c1_fixture("pure_svd_c1.npz")


@pytest.mark.parametrize("ev", ["host", "device"])
def test_run_experiment_matches_the_reference_run(c1, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / f"PureSVD_{ev}"
    res = c1h.run(out, synth_c1.pure_svd_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n"), ev == "device")
    c1h.assert_metrics(res, g["metrics"].tolist(), g["test_metrics"], "PureSVD", ev)
    if ev == "device":
        c1h.assert_no_rec_files(out)
        return
    files = sorted(os.listdir(out / "recs"))
    assert files == [str(g["rec_file"])], files                   # the reference's model name
    rec = np.loadtxt(out / "recs" / str(g["rec_file"]), delimiter="\t")
    users = np.unique(g["rec_users"])
    mine = rec[np.isin(rec[:, 0].astype(np.int64), users)]
    gu, gi, gs = g["rec_users"], g["rec_items"], g["rec_scores"]
    assert np.array_equal(np.unique(mine[:, 0]).astype(np.int64), users)
    k = 10
    scale = np.abs(gs).max()
    same = total = 0
    for u in users:
        a, b = mine[mine[:, 0] == u], (gu == u)
        ref_items, ref_scores = gi[b], gs[b]
        assert len(a) == len(ref_items) == k
        assert np.abs(a[:, 2] - ref_scores).max() <= 1e-3 * scale, u     # fp32 reference vs fp64 device
        iso = opsvd.isolated_abs(a[None, :, 2], np.array([-np.inf]), 1e-4 * scale)[0]
        iso[-1] = False                                                    # the k+1-th value is not in the file
        assert np.array_equal(a[iso, 1].astype(np.int64), ref_items[iso]), u
        same += iso.sum()
        total += k
    assert same > 0.5 * total, (same, total)
