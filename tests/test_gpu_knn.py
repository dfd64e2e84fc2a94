"""ItemKNN / UserKNN on the GPU: the exact bf16 Gram, the neighbour kernel (bit for bit against oracle/knn.py), the fused
sparse product + masked top-k, both models against the reference's goldens, and the reference's hello-world ItemKNN block
end to end at C1 scale."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, dev_csr
from elliot_b200 import ops, synth_c1
from elliot_b200.recommender import knn
from oracle import knn as oknn
from oracle.knn import isolated

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _int_matrix(U, I, dens, hi, seed):
    g = np.random.default_rng(seed)
    return np.where(g.random((U, I)) < dens, g.integers(1, hi + 1, (U, I)), 0).astype(np.float64)


# ---------------------------------------------------------------- 1. Gram exactness
GRAM_CASES = {
    "items_small": (300, 200, "items"),
    "users_small": (200, 300, "users"),
    "items_splitk": (4096, 100, "items"),     # 1 x 1 output tiles, K = 4096 users: split-K
    "users_splitk": (100, 4096, "users"),
}


def _gram_check(name):
    U, I, over = GRAM_CASES[name]
    R = _int_matrix(U, I, 0.3, 5, U + I)
    if over == "items":
        R[:, 0] = 63; R[:, 2] = 63                  # diagonal and off-diagonal 63^2 * 4096 = 16 257 024, just under 2^24
    else:
        R[0, :] = 63; R[2, :] = 63
    urm = dev_csr(R)
    X, rs, cs = ops.csr_to_dense_bf16(*urm, I, row_sq=True, col_sq=True)
    Ri = R.astype(np.int64)
    if over == "items":
        G = ops.gemm_bf16(X, X, I, I, U, a_rows_are_k=True, b_rows_are_k=True)
        want = Ri.T @ Ri
    else:
        G = ops.gemm_bf16(X, X, U, U, I)
        want = Ri @ Ri.T
    got = G.cpu().numpy()
    assert want.max() < 2 ** 24
    if max(U, I) == 4096:
        assert np.diag(want).max() > 2 ** 23
    assert np.array_equal(got.astype(np.int64), want) and np.all(got == np.round(got)), np.abs(got - want).max()
    assert np.array_equal(cs.cpu().numpy(), np.diag(Ri.T @ Ri).astype(np.float32))
    assert np.array_equal(rs.cpu().numpy(), np.diag(Ri @ Ri.T).astype(np.float32))


@pytest.mark.parametrize("name", sorted(GRAM_CASES))
def test_gram_is_exact_on_integer_ratings(name):
    _gram_check(name)


def test_gram_is_exact_with_split_k_off():
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_knn as t\n"
            "for n in sorted(t.GRAM_CASES): t._gram_check(n)\nprint('ok')") % (ROOT, os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, EB_GEMM_SPLITK="0"), capture_output=True, text=True,
                       cwd=ROOT)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


# ---------------------------------------------------------------- 2. neighbours, bit for bit
def _nbr_matrix(U, I, dens, kind, seed):
    R = _int_matrix(U, I, dens, 5, seed)
    if kind == "half":
        R = R * np.random.default_rng(seed + 1).choice([0.5, 1.0], R.shape)
    R[:, 1] = R[:, 0]                               # duplicate item: exact ties
    R[1, :] = R[0, :]                               # duplicate user
    R[:, 5] = 0; R[:, I - 1] = 0                    # items without ratings
    R[7, :] = 0                                     # a user without ratings
    return R


@pytest.mark.parametrize("over", ["items", "users"])
@pytest.mark.parametrize("cosine", [True, False])
@pytest.mark.parametrize("k", [1, 50, 1024])
@pytest.mark.parametrize("dens,kind", [(0.2, "int"), (0.01, "int"), (0.2, "half")])
def test_neighbours_equal_the_oracle_bitwise(over, cosine, k, dens, kind):
    U, I = (300, 1203) if over == "items" else (1203, 300)       # n not a multiple of 8, k above the nonzeros at 1 %
    R = _nbr_matrix(U, I, dens, kind, 5 + k)
    n = I if over == "items" else U
    idx, val = knn.neighbours(dev_csr(R), U, I, over, k, cosine, slab_rows=64)         # 19 slabs
    S = oknn.similarity(oknn.gram(R, over), cosine)
    oi, ov, oc = oknn.neighbours(S, k)
    assert np.array_equal(idx.cpu().numpy(), oi)
    assert np.array_equal(val.cpu().numpy().view(np.int32), ov.view(np.int32))
    assert n == idx.shape[0]
    if dens == 0.01 and k == 1024:
        assert oc.max() < k                                        # every list shorter than k: -1 / 0 padding checked


def test_neighbour_counts_and_slab_offset():
    R = _nbr_matrix(200, 131, 0.05, "int", 3)
    urm = dev_csr(R)
    X, _, cs = ops.csr_to_dense_bf16(*urm, 131, col_sq=True)
    j0, S = 40, 48
    C = ops.gemm_bf16(X[:, j0:], X, S, 131, 200, a_rows_are_k=True, b_rows_are_k=True)
    idx, val, cnt = ops.knn_neighbors(C, 131, j0, cs, 20)
    oi, ov, oc = oknn.neighbours(oknn.similarity(oknn.gram(R, "items"), True), 20)
    assert np.array_equal(cnt.cpu().numpy(), oc[j0:j0 + S])
    assert np.array_equal(idx.cpu().numpy(), oi[j0:j0 + S]) and np.array_equal(val.cpu().numpy(), ov[j0:j0 + S])


# ---------------------------------------------------------------- 3. fused score + top-k
def _score_case(n_rows, n_mid, n_cols, seed, integer):
    g = np.random.default_rng(seed)
    A = sp.random(n_rows, n_mid, density=0.05, random_state=seed, format="csr", dtype=np.float64)
    B = sp.random(n_mid, n_cols, density=min(1.0, 40.0 / n_cols + 0.002), random_state=seed + 1, format="csr", dtype=np.float64)
    if integer:
        A.data = g.integers(1, 6, A.nnz).astype(np.float64); B.data = g.integers(1, 4, B.nnz).astype(np.float64)
    else:
        A.data = A.data.astype(np.float32).astype(np.float64); B.data = B.data.astype(np.float32).astype(np.float64)
    A = A.tolil(); A[3, :] = 0; A = A.tocsr(); A.eliminate_zeros()          # a row without A entries
    mask = sp.random(n_rows, n_cols, density=0.1, random_state=seed + 2, format="csr")
    mask = mask.tolil()
    if n_cols > 3:
        mask[5, :] = 1; mask[5, n_cols - 1] = 0; mask[5, 1] = 0              # only two unmasked columns: -1 padding
    mask = sp.csr_matrix(mask); mask.data[:] = 1
    return A, B, mask


def _oracle_topk(A, B, mask, k, rows):
    P = (A @ B).toarray()
    M = mask.toarray() != 0
    return oknn.topk(P[rows], M[rows], k)


@pytest.mark.parametrize("n_cols", [1, 300, "tile", "tile+1"])
@pytest.mark.parametrize("k", [1, 10, 100])
def test_score_topk_integer_data_is_exact(n_cols, k):
    T = ops.knn_score_tile_cols()
    n_cols = {"tile": T, "tile+1": T + 1}.get(n_cols, n_cols)
    A, B, mask = _score_case(64, 50, n_cols, n_cols + k, integer=True)
    dA, dB, dM = dev_csr(A), dev_csr(B), dev_csr(mask)
    f = knn.frac_bits(knn._bound(dA, dB))
    idx, val = ops.knn_score_topk(dA, dB, n_cols, k, f, dM[0], dM[1])
    oi, ov = _oracle_topk(A, B, mask, k, np.arange(64))
    # integer sums below 2^24: exact, so the whole list is fixed, zero-score fill in column order and padding included
    assert np.array_equal(idx.cpu().numpy(), oi)
    assert np.array_equal(val.cpu().numpy(), ov.astype(np.float32))
    assert not np.any(mask.toarray()[np.arange(64)[:, None], np.maximum(oi, 0)] * (oi >= 0))
    idx2, val2 = ops.knn_score_topk(dA, dB, n_cols, k, f, dM[0], dM[1])
    assert torch.equal(idx, idx2) and torch.equal(val.view(torch.int32), val2.view(torch.int32))


@pytest.mark.parametrize("select", ["all", "users", "begin"])
@pytest.mark.parametrize("k", [10, 1024])
def test_score_topk_real_values_within_bound(select, k):
    n_cols = ops.knn_score_tile_cols() + 77
    A, B, mask = _score_case(96, 80, n_cols, 9 + k, integer=False)
    dA, dB, dM = dev_csr(A), dev_csr(B), dev_csr(mask)
    f = knn.frac_bits(knn._bound(dA, dB))
    if select == "users":
        rows = np.array([95, 3, 5, 40, 40, 0], np.int32)
        idx, val = ops.knn_score_topk(dA, dB, n_cols, k, f, dM[0], dM[1], users=torch.from_numpy(rows).to(DEV))
    elif select == "begin":
        rows = np.arange(17, 96)
        idx, val = ops.knn_score_topk(dA, dB, n_cols, k, f, dM[0], dM[1], user_begin=17, n_sel=len(rows))
    else:
        rows = np.arange(96)
        idx, val = ops.knn_score_topk(dA, dB, n_cols, k, f, dM[0], dM[1])
    P = (A @ B).toarray()[rows]
    oi, ov = _oracle_topk(A, B, mask, k, rows)
    gi, gv = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
    nterms = np.diff(A.indptr)[rows]                               # terms per output entry <= nonzeros of the A row
    with np.errstate(invalid="ignore"):
        tol = np.spacing(np.abs(ov).astype(np.float32)).astype(np.float64) + nterms[:, None] * 2.0 ** -(f + 1)
    filled = oi >= 0
    assert np.array_equal(gi >= 0, filled)
    assert np.all(np.abs(gv[filled] - ov[filled]) <= tol[filled])
    # the oracle's score of every returned column matches the oracle's value at that rank (sets equal up to ties)
    got_scores = np.where(filled, np.take_along_axis(P, np.maximum(gi, 0), 1), -np.inf)
    assert np.all(np.abs(got_scores[filled] - ov[filled]) <= 2 * tol[filled])
    # isolated ranks: the same column
    t2 = 2 * tol
    iso = filled.copy()
    with np.errstate(invalid="ignore"):
        iso[:, 1:] &= (ov[:, :-1] - ov[:, 1:]) > t2[:, 1:]
        iso[:, :-1] &= (ov[:, :-1] - ov[:, 1:]) > t2[:, :-1]
    assert np.array_equal(gi[iso], oi[iso])
    z = filled & (ov == 0)                                         # exact zeros: unmasked columns in ascending order
    assert np.array_equal(gi[z], oi[z])
    M = mask.toarray()[rows]
    assert not np.any((M[np.arange(len(rows))[:, None], np.maximum(gi, 0)] != 0) & filled)


# ---------------------------------------------------------------- 4. the models' pipeline against the reference's goldens
class _Data:
    def __init__(self, R):
        m = sp.csr_matrix(R.astype(np.float32))
        self.sp_i_train_ratings = m
        self.sp_i_train = sp.csr_matrix((np.ones(m.nnz, np.float32), m.indices, m.indptr), shape=m.shape)


def _isolated(v, v_next=None):
    """Ranks more than 2e-5 (relative) away from both neighbours; without the (k+1)-th values the last rank counts as
    isolated when it is from the previous one."""
    return isolated(v, np.full(len(v), -np.inf) if v_next is None else v_next)


@pytest.mark.parametrize("model", ["itemknn", "userknn"])
@pytest.mark.parametrize("size", ["tiny", "small"])
def test_models_match_reference_goldens(model, size):
    """The model's neighbour lists equal the oracle's bit for bit (the reference breaks exact ties at rank `neighbors`
    either way, oracle tests cover its lists); scored over the reference's own lists, the top-k lists equal the reference's
    at every isolated rank and the values agree within 1e-5."""
    g = dict(np.load(os.path.join(GOLD, f"{model}_{size}.npz")))
    over, k_nn, k = str(g["over"]), int(g["k_nn"]), int(g["topk"])
    for kind in ("int", "implicit", "half"):
        for sim in ("cosine", "dot"):
            tag = f"{kind}_{sim}"
            R = g[f"{tag}_R"]
            Ru = (R != 0).astype(np.float64) if kind == "implicit" else R
            m = knn.KNNModel(_Data(R), k_nn, sim, kind == "implicit", over, DEV)
            m.initialize()
            idx, val = knn.neighbours(m.urm, m.n_users, m.n_items, over, k_nn, sim == "cosine")
            oi, ov, _ = oknn.neighbours(oknn.similarity(oknn.gram(Ru, over), sim == "cosine"), k_nn)
            assert np.array_equal(idx.cpu().numpy(), oi) and np.array_equal(val.cpu().numpy(), ov), tag
            W = knn.transpose_lists(torch.from_numpy(g[f"{tag}_nbr_idx"]).to(DEV), torch.from_numpy(g[f"{tag}_nbr_val"]).to(DEV))
            m.A, m.B = (m.urm, W) if over == "items" else (W, m.urm)
            m.frac_bits = knn.frac_bits(knn._bound(m.A, m.B))
            mask = dev_csr(R != 0)
            ti, tv = m.topk(k, mask[0], mask[1])
            gi, gv = ti.cpu().numpy(), tv.cpu().numpy()
            ri, rv = g[f"{tag}_topk_idx"], g[f"{tag}_topk_val"]
            _, nv = oknn.topk(oknn.preds(Ru, g[f"{tag}_nbr_idx"], g[f"{tag}_nbr_val"], over), R != 0, k + 1)
            iso = _isolated(rv, nv[:, k])
            assert np.array_equal(gi[iso], ri[iso]), tag
            ok = np.isfinite(rv)
            assert np.array_equal(gi >= 0, ok), tag
            assert np.allclose(gv[ok], rv[ok], rtol=1e-5, atol=1e-6), tag


# ---------------------------------------------------------------- 5. the reference's hello world at C1 scale
c1 = c1h.c1_fixture("itemknn_c1.npz")


def test_hello_world_itemknn_matches_the_reference_run(c1):
    g, d, tsv = c1
    out = d / "host"
    res = c1h.run(out, synth_c1.hello_world_yaml(tsv, str(out)))
    c1h.assert_metrics(res, g["metrics"].tolist(), g["test_metrics"])
    files = os.listdir(out / "recs")
    assert files == [str(g["rec_file"])], (files, str(g["rec_file"]))
    rec = np.loadtxt(out / "recs" / files[0], delimiter="\t")
    users = np.unique(g["rec_users"])
    sel = np.isin(rec[:, 0].astype(np.int64), users)
    mine, ref = rec[sel], np.stack([g["rec_users"], g["rec_items"], g["rec_scores"]], 1)
    assert mine.shape == ref.shape
    mi, ri = mine[:, 1].reshape(len(users), -1), ref[:, 1].reshape(len(users), -1)
    rv = ref[:, 2].reshape(len(users), -1)
    iso = _isolated(rv)
    assert (iso & (mi == ri)).mean() >= 0.95, ((iso & (mi == ri)).mean(), iso.mean())
    assert np.allclose(mine[:, 2].reshape(rv.shape)[iso & (mi == ri)], rv[iso & (mi == ri)], rtol=1e-5)


def test_hello_world_itemknn_device_eval_without_recs(c1):
    g, d, tsv = c1
    out = d / "device"
    res = c1h.run(out, synth_c1.hello_world_yaml(tsv, str(out), model_extra="      b200_eval: device\n"), device_eval=True)
    c1h.assert_metrics(res, g["metrics"].tolist(), g["test_metrics"])
    c1h.assert_no_rec_files(out)
