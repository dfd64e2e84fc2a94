"""RP3beta on the GPU: the similarity lists, W and the scores against the oracle and the reference's goldens bit for bit,
reruns, the column-tiled path on a catalogue wider than one shared-memory row, and the reference's run_experiment on
recsys_config.yml's RP3beta block at C1 scale."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, all_scores, to_dev, w_host
from elliot_b200 import ops
from elliot_b200._lib import EbError
from oracle import rp3beta as orp3
from oracle.knn import isolated, topk as oracle_topk

pytestmark = pytest.mark.gpu
_G = dict(np.load(os.path.join(GOLD, "rp3beta_cases.npz")))


def _dev_csr(M):
    return c1h.dev_csr(M, sort=False)


class _Data:
    def __init__(self, R):
        self.sp_i_train_ratings = R if sp.issparse(R) else sp.csr_matrix(R.astype(np.float32))


def _case(name):
    R = _G[f"{name}_R"].astype(np.float64)
    nbh = int(_G[f"{name}_neighborhood"])
    return (R, float(_G[f"{name}_alpha"]), float(_G[f"{name}_beta"]), bool(_G[f"{name}_normalize"]),
            R.shape[1] if nbh == -1 else nbh)


def _device_lists(m):
    (pp, pi, pv), (qp, qi, qv), degree = m.host_operands()
    idx, val, cnt = ops.rp3_similarity((to_dev(qp, torch.int64), to_dev(qi, torch.int32), to_dev(qv)),
                                       (to_dev(pp, torch.int64), to_dev(pi, torch.int32), to_dev(pv)), to_dev(degree, torch.float64), m.k)
    idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
    return {i: (idx[i, :cnt[i]].astype(np.int64), val[i, :cnt[i]]) for i in range(len(cnt))}


# ---------------------------------------------------------------- 1. the model against the oracle and the goldens
@pytest.mark.parametrize("name", list(_G["cases"]))
def test_similarity_w_and_scores_match(name):
    from elliot_b200.recommender.rp3beta import RP3Model
    R, alpha, beta, norm, k = _case(name)
    n = R.shape[1]
    data = _Data(R)
    before = [a.tobytes() for a in (data.sp_i_train_ratings.data, data.sp_i_train_ratings.indices,
                                    data.sp_i_train_ratings.indptr)]
    m = RP3Model(data, int(_G[f"{name}_neighborhood"]), alpha, beta, norm, DEV)
    W_or, lists_or = orp3.weights(data.sp_i_train_ratings, alpha, beta, k, norm)
    # every similarity row: the same columns and bit-equal values as the oracle (same tie rule)
    mine = _device_lists(m)
    for i in range(n):
        assert np.array_equal(mine[i][0], lists_or[i][0]), (name, i)
        assert np.array_equal(mine[i][1].view(np.int32), lists_or[i][1].view(np.int32)), (name, i)
    m.initialize()
    W = w_host(m.W, n)
    assert np.array_equal(W.indptr, W_or.indptr) and np.array_equal(W.indices, W_or.indices), name
    assert np.array_equal(W.data.view(np.int32), W_or.data.view(np.int32)), name
    ref_lists = orp3.reference_lists(_G[f"{name}_s_row"], _G[f"{name}_s_col"], _G[f"{name}_s_val"], n)
    W_ref = sp.csc_matrix((_G[f"{name}_w_data"], _G[f"{name}_w_rows"], _G[f"{name}_w_ptr"]), shape=(n, n)).tocsr()
    orp3.w_equal_but_ties(W, W_ref, lists_or, ref_lists, k)
    # scores from the golden's own W: bit-equal to the reference's preds
    W_ref.sort_indices()
    P = all_scores(m.urm, _dev_csr(W_ref), n)
    assert orp3.preds_digest(P) == str(_G[f"{name}_preds_sha256"]), name
    # the model's lists equal the oracle's (same W, same tie rule), and with the golden's W the reference's lists
    # wherever the k-th and (k+1)-th scores differ
    K = int(_G["topk"])
    mask = _dev_csr(R != 0)
    ti, tv = m.topk(K, mask[0], mask[1])
    gi, gv = ti.cpu().numpy(), tv.cpu().numpy()
    oi, ov = oracle_topk(orp3.preds(data.sp_i_train_ratings, W_or).astype(np.float64), R != 0, K)
    assert np.array_equal(gi, oi), name
    assert np.array_equal(gv.astype(np.float64)[gi >= 0], ov[gi >= 0]), name
    ri, _ = ops.rp3_score_topk(m.urm, _dev_csr(W_ref), n, K, mask[0], mask[1])
    _, rv = oracle_topk(P.astype(np.float64), R != 0, K + 1)
    iso = isolated(rv[:, :K], rv[:, K], rel=0.0)
    assert np.array_equal(ri.cpu().numpy()[iso], _G[f"{name}_topk_idx"][iso]), name
    after = [a.tobytes() for a in (data.sp_i_train_ratings.data, data.sp_i_train_ratings.indices,
                                   data.sp_i_train_ratings.indptr)]
    assert before == after, "the DataSet must not change"


def test_neighborhood_minus_one_keeps_every_nonzero():
    from elliot_b200.recommender.rp3beta import RP3Model
    name = "implicit_a0.5_b0_nbm1"
    R, alpha, beta, norm, k = _case(name)
    m = RP3Model(_Data(R), -1, alpha, beta, norm, DEV)
    assert m.k == R.shape[1]
    m.initialize()
    W_or, _ = orp3.weights(sp.csr_matrix(R.astype(np.float32)), alpha, beta, k, norm)
    W = w_host(m.W, R.shape[1])
    assert W.nnz == W_or.nnz == int(_G[f"{name}_w_data"].size)


def test_reruns_are_bit_identical():
    from elliot_b200.recommender.rp3beta import RP3Model
    R, alpha, beta, norm, k = _case("half_a1.0807_b0.6_norm_nbm1")
    mask = _dev_csr(R != 0)
    outs = []
    for _ in range(2):
        m = RP3Model(_Data(R), k, alpha, beta, norm, DEV)
        m.initialize()
        ti, tv = m.topk(50, mask[0], mask[1])
        outs.append([a.cpu().numpy().view(np.int32) for a in (*m.W[1:], ti, tv)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


# ---------------------------------------------------------------- 2. wider than one shared-memory row
def test_column_tiled_path_matches_the_oracle():
    T = ops.rp3_tile_cols()
    n, U = T + 8000, 700
    g = np.random.default_rng(21)
    rows, cols = [], []
    for u in range(U):
        c = g.choice(n, size=int(g.integers(3, 60)), replace=False)
        c[:3] = [0, T - 1, n - 1] if u % 7 == 0 else c[:3]          # columns on both sides of the tile edge
        c = np.unique(c)
        rows.append(np.full(len(c), u)); cols.append(c)
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    R = sp.csr_matrix((g.integers(1, 11, rows.size) / 2.0, (rows, cols)), shape=(U, n), dtype=np.float32)
    from elliot_b200.recommender.rp3beta import RP3Model
    m = RP3Model(_Data(R), 25, 1.0807, 0.7029, True, DEV)
    mine = _device_lists(m)
    Pui, Piu, degree = orp3.prepare(R, 1.0807, 0.7029)
    sample = np.unique(np.concatenate([[0, T - 1, T, n - 1], g.choice(n, 60, replace=False)]))
    want = orp3.similarity_lists(Pui, Piu, degree, 25, rows=sample)
    for i in sample:
        assert np.array_equal(mine[i][0], want[i][0]), i
        assert np.array_equal(mine[i][1].view(np.int32), want[i][1].view(np.int32)), i
    # scoring over a random W of the same width, with a mask
    W = sp.random(n, n, density=3e-5, format="csr", dtype=np.float32, random_state=4)
    W.data = (g.random(W.nnz) * 1e-2).astype(np.float32)
    W.sort_indices()
    users = np.array([0, 7, 14, 350, 699, 3], np.int32)
    mask = _dev_csr(R != 0)
    ti, tv = ops.rp3_score_topk(m.urm, _dev_csr(W), n, 100, mask[0], mask[1], users=to_dev(users))
    P = orp3.preds(R, W, rows=users).astype(np.float64)
    oi, ov = oracle_topk(P, (R != 0).toarray()[users], 100)
    assert np.array_equal(ti.cpu().numpy(), oi)
    assert np.array_equal(tv.cpu().numpy().astype(np.float64), ov)


def test_bad_arguments_are_refused():
    A = _dev_csr(sp.eye(4))
    with pytest.raises(EbError, match="k=1025"):
        ops.rp3_score_topk(A, A, 4, 1025)


# ---------------------------------------------------------------- 3. run_experiment at C1 scale
c1 = c1h.c1_fixture("rp3beta_c1.npz")


@pytest.mark.parametrize("ev", ["host", "device"])
def test_run_experiment_matches_the_reference_run(c1, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / ev
    res = c1h.run(out, synth_c1.rp3beta_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n"), ev == "device")
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
    assert np.array_equal(mine[:, 2].astype(np.float32), g["rec_scores"].astype(np.float32))
