"""SLIM on the GPU: every item's coefficients, epoch counts and W against the oracle and the reference's goldens, the
scores from the golden's W against the reference's preds bit for bit, the global-residual path against the
shared-memory one, reruns, the shape the reference cannot fit, and the reference's run_experiment on
recsys_config.yml's Slim block at C1 scale."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import c1_harness as c1h
from c1_harness import DEV, GOLD, all_scores, dev_csr, w_host
from oracle import slim as oslim
from oracle.knn import isolated, topk as oracle_topk
from oracle.rp3beta import preds_digest

pytestmark = pytest.mark.gpu
_G = dict(np.load(os.path.join(GOLD, "slim_cases.npz")))


class _Data:
    def __init__(self, R):
        self.sp_i_train_ratings = sp.csr_matrix(R.astype(np.float32))


def _model(name, **kw):
    from elliot_b200.recommender.slim import SlimModel
    R = _G[f"{name}_R"].astype(np.float32)
    m = SlimModel(_Data(R), float(_G[f"{name}_l1_ratio"]), float(_G[f"{name}_alpha"]), int(_G[f"{name}_neighborhood"]),
                  int(_G["seed"]), DEV)
    m.initialize(**kw)
    return R, m


# ---------------------------------------------------------------- 1. the model against the oracle and the goldens
@pytest.mark.parametrize("name", list(_G["cases"]))
def test_coefficients_w_and_scores_match(name):
    R, m = _model(name)
    n = R.shape[1]
    coef = m.coef_t.cpu().numpy().T.copy()
    n_iter = m.n_iter.cpu().numpy()
    # coefficients within 1e-5 of each item's largest, equal epochs, W equal but ties, the golden's preds and lists
    oslim.check_case(_G, name, coef=coef, n_iter=n_iter)
    # against the oracle: the same float32 updates, so the same bits
    oc, oi, og = oslim.fit(R, float(_G[f"{name}_alpha"]), float(_G[f"{name}_l1_ratio"]), int(_G["seed"]))
    assert np.array_equal(coef.view(np.int32), oc.view(np.int32)), name
    assert np.array_equal(n_iter, oi), name
    assert np.allclose(m.gap.cpu().numpy(), og, rtol=1e-3, atol=1e-12), name
    assert np.array_equal(m.nnz.cpu().numpy(), (oc != 0).sum(1)), name
    W = w_host(m.W, n)
    W_or = oslim.select(oc, int(_G[f"{name}_neighborhood"]))
    assert np.array_equal(W.indptr, W_or.indptr) and np.array_equal(W.indices, W_or.indices), name
    assert np.array_equal(W.data.view(np.int32), W_or.data.view(np.int32)), name
    Wg = oslim.golden_W(_G, name)
    oslim.w_equal_except_ties(W, Wg, _G[f"{name}_coef"])
    # scores from the golden's own W: bit-equal to the reference's preds
    Wg.sort_indices()
    P = all_scores(m.urm, dev_csr(Wg), n)
    assert preds_digest(P) == str(_G[f"{name}_preds_sha256"]), name
    # the model's lists: the oracle's, and the reference's at isolated ranks
    K = int(_G["topk"])
    mask = dev_csr(R != 0)
    ti, tv = m.topk(K, mask[0], mask[1])
    gi = ti.cpu().numpy()
    oi_, ov_ = oracle_topk(oslim.preds(R, W_or).astype(np.float64), R != 0, K + 1)
    assert np.array_equal(gi, oi_[:, :K]), name
    iso = isolated(ov_[:, :K], ov_[:, K], rel=0.0)
    assert np.array_equal(gi[iso], _G[f"{name}_topk_idx"][iso]), name


def test_global_residual_path_equals_the_shared_one():
    for name in ("int_tois", "half_screen"):
        outs = []
        for shared, slots in ((True, None), (False, None), (False, 7)):
            _, m = _model(name, shared_residual=shared, slots=slots)
            outs.append([a.cpu().numpy().view(np.int32) for a in (m.coef_t, m.n_iter, m.gap, *m.W[1:])])
        for o in outs[1:]:
            for a, b in zip(outs[0], o):
                assert np.array_equal(a, b), name


def test_reruns_are_bit_identical():
    outs = []
    for _ in range(2):
        R, m = _model("implicit_default")
        mask = dev_csr(R != 0)
        ti, tv = m.topk(50, mask[0], mask[1])
        outs.append([a.cpu().numpy().view(np.int32) for a in (m.coef_t, m.n_iter, *m.W[1:], ti, tv)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_more_items_than_users_is_refused():
    from elliot_b200.recommender.slim import SlimModel
    with pytest.raises(ValueError, match="num_items <= num_users"):
        SlimModel(_Data(np.ones((3, 5))), 0.5, 0.05, 10, 42, DEV)


# ---------------------------------------------------------------- 2. run_experiment at C1 scale
c1 = c1h.c1_fixture("slim_c1.npz")


@pytest.mark.parametrize("ev", ["host", "device"])
def test_run_experiment_matches_the_reference_run(c1, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / ev
    res = c1h.run(out, synth_c1.slim_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n"), ev == "device")
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
