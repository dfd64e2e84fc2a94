"""GPU tests of ConvNeuMF (csrc/convneumf.cu, recommender/convneumf.py): the level-1 kernels, the head and whole steps
(loss and every parameter after Keras Adam) against the fp64 restatements of oracle/convneumf.py in the exact_gemm
checking mode and on the bf16 tensor-core path, chunked against unchunked batches, dropout, the fused scorer against fp64
scores and against itself, top-k, the dense rank pass, C1 runs through run_experiment, and the refusals."""
import numpy as np
import pytest
import torch
import yaml

from elliot_b200 import ops, synth_c1
from oracle import auc as auc_oracle
from oracle import convneumf as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32, UBF = 2.0 ** -24, 2.0 ** -8


def _model(f, widths, nu, ni, p_drop=0.0, l_w=0.005, seed=3):
    from elliot_b200.recommender.convneumf import ConvNeuMFModel
    return ConvNeuMFModel(nu, ni, f, 1e-3, widths, p_drop, l_w, 0.0005, seed, DEV)


def _load(m, P, U, I):
    """Oracle parameters (Keras shapes) and tables into the device model."""
    f, L = m.f, m.L
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float().to(DEV)
    m.P["U"].zero_(); m.P["U"][:, :f] = t(U)
    m.P["I"].zero_(); m.P["I"][:, :f] = t(I)
    m.P["W1"].copy_(t(P["W1"].reshape(-1))); m.P["b1"].copy_(t(P["b1"]))
    for l in range(2, L + 1):
        K = P["K"][l]
        m.P[f"W{l}"].copy_(t(K.reshape(-1, K.shape[3]).T)); m.P[f"b{l}"].copy_(t(P["b"][l]))
    m.P["Wd1"].copy_(t(P["Wd1"].reshape(-1))); m.P["bd1"].copy_(t(P["bd1"])); m.P["wd2"].copy_(t(P["wd2"]))
    m.P["bd2"].zero_(); m.P["bd2"][0] = float(P["bd2"][0])
    m._refresh()


def _grads_host(m):
    """The device gradients in the oracle's shapes."""
    f, L, G = m.f, m.L, m.G
    h = lambda t: t.double().cpu().numpy()
    out = {"W1": h(G["W1"]).reshape(2, 2, 1, -1), "b1": h(G["b1"]), "K": [None, None], "b": [None, None],
           "Wd1": h(G["Wd1"]).reshape(m.c[L], m.c[L]), "bd1": h(G["bd1"]), "wd2": h(G["wd2"]), "bd2": h(G["bd2"])[:1]}
    for l in range(2, L + 1):
        out["K"].append(h(G[f"W{l}"]).T.reshape(2, 2, m.c[l - 1], m.c[l])); out["b"].append(h(G[f"b{l}"]))
    return out, h(G["U"])[:, :f], h(G["I"])[:, :f]


def _case(rs, f, widths, nu, ni, B, scale=1.0):
    P = oracle.init_params(rs, widths)
    U = rs.uniform(-scale, scale, (nu, f)).astype(np.float32).astype(np.float64)
    I = rs.uniform(-scale, scale, (ni, f)).astype(np.float32).astype(np.float64)
    P = {k: ([None if a is None else a.astype(np.float32).astype(np.float64) for a in v] if isinstance(v, list)
             else v.astype(np.float32).astype(np.float64)) for k, v in P.items()}
    tu = rs.randint(0, nu, B).astype(np.int32); ti = rs.randint(0, ni, B).astype(np.int32)
    tj = rs.randint(0, ni, B).astype(np.int32)
    tu[: B // 4] = tu[0]; ti[: B // 8] = ti[0]                         # repeated users and items
    return P, U, I, tu, ti, tj


def _flat(G, dU, dI):
    parts = [G["W1"], G["b1"], G["Wd1"], G["bd1"], G["wd2"], G["bd2"], dU, dI]
    parts += [a for a in G["K"][2:]] + [a for a in G["b"][2:]]
    return parts


def _close(got, want, rel, B):
    """Every gradient within rel of its own tensor's largest magnitude, plus a floor for the sums over the batch's 2 B
    pairs that cancel (bd1 and bd2 add +g and -g per triple, exactly 0 in fp64): the fp32 reduction error of 2 B terms
    of magnitude <= 1, 4 u (2 B)^1.5."""
    floor = 4 * U32 * (2 * B) ** 1.5
    for g, w in zip(_flat(*got), _flat(*want)):
        tol = rel * np.abs(w).max() + floor
        assert np.abs(g - w).max() <= tol, (np.abs(g - w).max(), tol, w.shape)


def _device_step(m, tu, ti, tj, chunk=None):
    t = lambda a: torch.from_numpy(a).to(DEV)
    m._loss.zero_()
    m.grads(t(tu), t(ti), t(tj), chunk=chunk)
    torch.cuda.synchronize()
    return float(m._loss.item())


CASES = [(8, [8], 8, 12, 4096), (8, [8, 16], 10, 14, 1024), (100, [32, 32], 20, 30, 64), (101, [8, 32, 64], 12, 16, 32),
         (64, [16, 24, 8], 9, 11, 96), (256, [64, 8], 4, 5, 8)]


@pytest.mark.parametrize("f,widths,nu,ni,B", CASES)
@pytest.mark.parametrize("exact", [True, False])
def test_step_matches_fp64(f, widths, nu, ni, B, exact):
    """Loss and every gradient of one batch, then every parameter after one Keras Adam step.  exact_gemm: the levels
    >= 2 run the fp32 checking GEMM, so the step is fp32 throughout (bound ~ 1e-4 of each tensor's scale after
    accumulation over a batch, whose sums of up to 2 B R_1 terms cancel: 1e-3); bf16: every operand of a level is rounded
    to bf16, 2^-8 relative, in dot products of up to K = 4 c terms, and the error compounds over the L levels and the
    head: 2^-8 sqrt(K_max) (L + 1)."""
    rs = np.random.RandomState(f * 7 + len(widths) + B)
    P, U, I, tu, ti, tj = _case(rs, f, widths, nu, ni, B)
    with ops.exact_gemm(exact):
        m = _model(f, widths, nu, ni)
        _load(m, P, U, I)
        loss = _device_step(m, tu, ti, tj)
    want = oracle.loss_and_grads(P, U, I, tu, ti, tj, 0.005)
    rel = 1e-3 if exact else UBF * np.sqrt(4 * max(widths)) * (len(widths) + 1)
    assert loss == pytest.approx(want[0], rel=rel, abs=1e-3)
    _close(_grads_host(m), (want[1], want[2], want[3]), rel, B)
    if exact:
        with ops.exact_gemm(True):
            m.adam()
        opt = oracle.KerasAdam(1e-3)
        Uc, Ic = U.copy(), I.copy()
        oracle.adam_step(opt, P, Uc, Ic, want[1], want[2], want[3])
        # the first Adam step moves an element by lr g / (|g| + eps'): +-lr where |g| >> eps, but a gradient near eps moves
        # it by an amount its fp32 error changes; bound 5 % of lr
        for got, ref in ((m.P["U"][:, :f], Uc), (m.P["I"][:, :f], Ic), (m.P["W1"], P["W1"].reshape(-1)),
                         (m.P["Wd1"], P["Wd1"].reshape(-1))):
            assert np.abs(got.double().cpu().numpy() - ref).max() < 5e-5


def test_coordinates_beyond_m_get_only_the_regulariser():
    f, widths = 13, [8, 16]                                             # m = 12: coordinate 12 reaches no layer
    rs = np.random.RandomState(5)
    P, U, I, tu, ti, tj = _case(rs, f, widths, 6, 7, 64)
    with ops.exact_gemm(True):
        m = _model(f, widths, 6, 7, l_w=0.01)
        _load(m, P, U, I)
        _device_step(m, tu, ti, tj)
    _, dU, dI = _grads_host(m)
    cu = np.bincount(tu, minlength=6); ci = np.bincount(np.concatenate([ti, tj]), minlength=7)
    assert np.allclose(dU[:, 12], 0.01 * cu * U[:, 12], rtol=1e-5, atol=1e-7)
    assert np.allclose(dI[:, 12], 0.01 * ci * I[:, 12], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("exact", [True, False])
def test_chunked_batch_equals_unchunked(exact):
    f, widths, B = 32, [16, 16], 300
    rs = np.random.RandomState(11)
    P, U, I, tu, ti, tj = _case(rs, f, widths, 30, 40, B)
    got = []
    for chunk in (None, 64):
        with ops.exact_gemm(exact):
            m = _model(f, widths, 30, 40)
            _load(m, P, U, I)
            loss = _device_step(m, tu, ti, tj, chunk=chunk)
        got.append((loss, _grads_host(m)))
    assert got[1][0] == pytest.approx(got[0][0], rel=1e-9)
    _close(got[1][1], got[0][1], 1e-5, B)                              # only the order of the sums differs


def test_dropout_identity_rate_and_scale():
    f, widths, B = 16, [8, 32], 4096
    rs = np.random.RandomState(2)
    P, U, I, tu, ti, tj = _case(rs, f, widths, 50, 60, B)
    t = lambda a: torch.from_numpy(a).to(DEV)
    for p in (0.0, 0.3):
        with ops.exact_gemm(True):
            m = _model(f, widths, 50, 60, p_drop=p)
            _load(m, P, U, I)
            masks = torch.zeros((B, 2, 2, 32), device=DEV)
            y = torch.zeros(2 * B, device=DEV)
            m.grads(t(tu), t(ti), t(tj), y_out=y, mask_out=masks)
        mk = masks.cpu().numpy().astype(np.float64)
        if p == 0:
            assert np.all(mk == 1.0)
        else:
            kept = mk > 0
            assert abs(kept.mean() - 0.7) < 0.01
            assert np.all(np.abs(mk[kept] - 1 / 0.7) < 1e-6)
        # the step with these masks is the oracle's with the same masks
        want = oracle.loss_and_grads(P, U, I, tu, ti, tj, 0.005, masks=(mk[:, 0, 0], mk[:, 0, 1], mk[:, 1, 0], mk[:, 1, 1]))
        yv = y.cpu().numpy()
        assert np.abs(yv[:B] - want[4][0]).max() < 1e-4 * (np.abs(want[4][0]).max() + 1)
        _close(_grads_host(m), (want[1], want[2], want[3]), 1e-4, B)


SCORE_CASES = [(8, [8]), (100, [32, 32]), (101, [8, 32, 64]), (64, [16, 24, 8]), (256, [64, 8]), (40, [40, 56]), (48, [64, 16, 16])]


def _scorer_case(f, widths, nu, ni, seed):
    rs = np.random.RandomState(seed)
    P, U, I, *_ = _case(rs, f, widths, nu, ni, 1)
    m = _model(f, widths, nu, ni)
    _load(m, P, U, I)
    return m, P, U, I


@pytest.mark.parametrize("f,widths", SCORE_CASES)
def test_scorer_matches_fp64_and_reruns_bit_identical(f, widths):
    """Bound: level 1 and every level's output are rounded to bf16 (2^-8 relative) and the weights too; the error of a
    score stays below 3e-2 of the block's largest |score| + its spread."""
    nu, ni = (5, 77) if f < 256 else (2, 40)
    m, P, U, I = _scorer_case(f, widths, nu, ni, f + len(widths))
    got = m.scores(0, nu)
    again = m.scores(0, nu)
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    want = oracle.full_scores(P, U, I)
    g = got.double().cpu().numpy()
    scale = np.abs(want).max() + want.std()
    assert np.abs(g - want).max() <= 3e-2 * scale, (np.abs(g - want).max(), scale)
    # a user block other than the first gives the same rows
    part = m.scores(1, nu)
    assert torch.equal(part, got[1:])


def test_topk_near_ties_and_no_train_items():
    f, widths, nu, ni, k = 40, [16, 16], 30, 500, 10
    m, P, U, I = _scorer_case(f, widths, nu, ni, 9)
    rs = np.random.RandomState(1)
    rows = [np.sort(rs.choice(ni, rs.randint(0, 40), replace=False)) for _ in range(nu)]
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    ind = np.concatenate(rows).astype(np.int32)
    idx, val = m.topk(k, torch.from_numpy(indptr).to(DEV), torch.from_numpy(ind).to(DEV))
    idx, val = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
    S = oracle.full_scores(P, U, I)
    tol = 3e-2 * (np.abs(S).max() + S.std())
    for u in range(nu):
        s = S[u].copy(); s[rows[u]] = -np.inf
        kth = np.sort(s)[::-1][k - 1]
        assert not set(idx[u]) & set(rows[u].tolist())
        assert np.all(s[idx[u]] >= kth - 2 * tol)                      # listed items are the k best up to near-ties
        assert np.all(np.abs(val[u] - S[u, idx[u]]) <= tol)
        assert np.all(np.diff(val[u]) <= 0)


def _rel_csr(rs, nu, ni, extra_outside=True):
    rows = [np.sort(rs.choice(ni, rs.randint(0, 30), replace=False)).astype(np.int32) for _ in range(nu)]
    if extra_outside:
        rows[0] = np.concatenate([[-1], rows[0]]).astype(np.int32)
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    return rows, torch.from_numpy(indptr).to(DEV), torch.from_numpy(np.concatenate(rows).astype(np.int32)).to(DEV)


def test_dense_rank_equals_score_rank_on_a_factor_block():
    """Small integer factors: every dot product is exact in fp32, so the dense U.V^T block holds score_rank's own scores
    (ties included)."""
    rs = np.random.RandomState(4)
    nu, ni, d = 40, 700, 16
    U = rs.randint(-2, 3, (nu, d)).astype(np.float32); V = rs.randint(-2, 3, (ni, d)).astype(np.float32)
    Ut, Vt = torch.from_numpy(U).to(DEV), torch.from_numpy(V).to(DEV)
    rel, rp, ri = _rel_csr(rs, nu, ni)
    mrows, mp, mi = _rel_csr(rs, nu, ni, extra_outside=False)
    want = ops.score_rank(Ut, Vt, None, d, rp, ri, mp, mi)
    S = torch.from_numpy(U.astype(np.float64) @ V.T.astype(np.float64)).float().to(DEV)
    S[3, 5] = float("nan"); S[4, 6] = float("-inf")
    got = ops.dense_rank(S, rp, ri, mp, mi)
    # rows 3 and 4 differ from the factor block by one unlisted entry: compare the others, and those on the host
    for a, b in zip(got, want):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        keep = np.ones(nu, bool); keep[[3, 4]] = False
        assert np.array_equal(a[keep], b[keep])
    Sh = S.cpu().numpy()
    for u in (3, 4):
        s = Sh[u].copy(); s[mrows[u]] = -np.inf
        ok = np.isfinite(s)
        order = sorted(np.nonzero(ok)[0], key=lambda j: (-s[j], j))
        c = auc_oracle.rank_counts([int(j) for j in order], [int(j) for j in rel[u] if j >= 0])
        assert (int(got[0][u]), int(got[1][u])) == c[:2]


def test_dense_rank_on_scorer_output_equals_host_count():
    f, widths, nu, ni = 32, [8, 16], 12, 300
    m, *_ = _scorer_case(f, widths, nu, ni, 21)
    rs = np.random.RandomState(8)
    rel, rp, ri = _rel_csr(rs, nu, ni)
    mrows, mp, mi = _rel_csr(rs, nu, ni, extra_outside=False)
    n_pos, sum_c = m.rank(rp, ri, mp, mi)
    S = m.scores(0, nu).cpu().numpy()
    for u in range(nu):
        s = S[u].copy(); s[mrows[u]] = -np.inf
        order = sorted(np.nonzero(np.isfinite(s))[0], key=lambda j: (-s[j], j))
        c = auc_oracle.rank_counts([int(j) for j in order], [int(j) for j in rel[u] if j >= 0])
        assert (int(n_pos[u]), int(sum_c[u])) == c[:2], u


# ---------------------------------------------------------------- refusals
@pytest.mark.parametrize("kw,err,match", [
    ({"cnn_kernels": [3, 2]}, NotImplementedError, "kernels and strides of 2"),
    ({"cnn_strides": [2, 1]}, NotImplementedError, "kernels and strides of 2"),
    ({"cnn_channels": [1, 32, 12]}, ValueError, "multiple of 8"),
    ({"cnn_channels": [1, 32, 72]}, ValueError, "multiple of 8"),
    ({"cnn_channels": [1, 32]}, RuntimeError, "don't match"),
    ({"cnn_kernels": [2, 2, 2]}, RuntimeError, "don't match"),
    ({"embedding_size": 3}, ValueError, "2\\^2 <= embedding_size"),
    ({"embedding_size": 300}, ValueError, "<= 256"),
    ({"embedding_size": 256, "cnn_channels": [1] + [64] * 8, "cnn_kernels": [2] * 8, "cnn_strides": [2] * 8}, ValueError,
     "shared memory"),
])
def test_config_refusals(kw, err, match):
    from elliot_b200.recommender.convneumf import check_config
    args = {"embedding_size": 100, "cnn_channels": [1, 32, 32], "cnn_kernels": [2, 2], "cnn_strides": [2, 2], **kw}
    with pytest.raises(err, match=match):
        check_config(args["embedding_size"], args["cnn_channels"], args["cnn_kernels"], args["cnn_strides"])


# ---------------------------------------------------------------- C1 runs through run_experiment
@pytest.fixture(scope="module")
def c1_tsv(tmp_path_factory):
    tsv = str(tmp_path_factory.mktemp("convneumf_c1") / "dataset.tsv")
    synth_c1.write_tsv(tsv)
    return tsv


def _c1_yaml(tsv, out, block, meta, metrics=("nDCG", "AUC", "GAUC"), extra=None):
    cfg = yaml.safe_load(synth_c1.experiment_yaml(tsv, out, "ConvNeuMF", "", metrics=metrics, meta=()))
    cfg["experiment"]["models"]["ConvNeuMF"] = dict(block, meta=meta)
    cfg["experiment"].update(extra or {})
    return yaml.safe_dump(cfg)


BLOCK = {"epochs": 2, "batch_size": 512, "embedding_size": 32, "cnn_channels": "(1, 16, 16)", "cnn_kernels": "(2,2)",
         "cnn_strides": "(2,2)", "lr": 0.001, "l_w": 0.005, "l_b": 0.0005, "dropout_prob": 0, "seed": 7}


def test_c1_run_device_and_host_metrics_agree_and_restore(c1_tsv, tmp_path):
    """Two epochs at batch 512 with nDCG, AUC and GAUC; the saved weights restored twice, once evaluated on the host
    and once on the device: the same scores (the scorer is deterministic), so the same lists and metrics, and the ones
    of the trained model's epoch whose weights were saved."""
    from elliot_b200 import run_experiment
    from elliot_b200.recommender import convneumf
    lists, models = [], []
    orig_topk, orig_train = convneumf.ConvNeuMFModel.topk, convneumf.ConvNeuMF.train

    def recording_topk(self, *a, **kw):
        out = orig_topk(self, *a, **kw)
        lists.append(tuple(t.cpu().numpy() for t in out))
        return out

    def recording_train(self):
        models.append(self)
        return orig_train(self)
    convneumf.ConvNeuMFModel.topk, convneumf.ConvNeuMF.train = recording_topk, recording_train
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), BLOCK, {"save_weights": True, "save_recs": False}))
        trained = run_experiment(str(p))[0]
        n_trained = len(lists)
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), BLOCK, {"restore": True, "save_recs": False}))
        host = run_experiment(str(p))[0]["test_results"][10]
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), dict(BLOCK, b200_eval="device"), {"restore": True, "save_recs": False}))
        dev = run_experiment(str(p))[0]["test_results"][10]
    finally:
        convneumf.ConvNeuMFModel.topk, convneumf.ConvNeuMF.train = orig_topk, orig_train
    assert trained["name"].startswith("ConvNeuMF_") and "cnn_channels=1-16-16" in trained["name"]
    assert len(trained["history"]) == 2
    assert all(np.isfinite(models[0]._losses))
    best = trained["test_results"][10]
    for name in ("nDCG", "AUC", "GAUC"):
        assert np.isfinite(best[name]) and host[name] == best[name], name
        assert dev[name] == pytest.approx(host[name], abs=1e-12), name
    assert best["AUC"] > 0.6                                           # two epochs learn a ranking better than chance
    assert np.array_equal(lists[-1][0], lists[-2][0]) and np.array_equal(lists[-1][1], lists[-2][1])
    assert any(np.array_equal(lists[-1][0], a) and np.array_equal(lists[-1][1], b) for a, b in lists[:n_trained])


def test_c1_rating_metrics_and_negative_sampling_refused_before_training(c1_tsv, tmp_path):
    from elliot_b200 import run_experiment
    from elliot_b200.recommender import convneumf
    trained = []
    orig = convneumf.ConvNeuMF.train
    convneumf.ConvNeuMF.train = lambda self: trained.append(1)
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), dict(BLOCK, epochs=1), {"save_recs": False}, metrics=("nDCG", "MAE")))
        with pytest.raises(Exception, match="ConvNeuMF cannot evaluate MAE"):
            run_experiment(str(p))
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), dict(BLOCK, epochs=1), {"save_recs": False}, metrics=("nDCG",),
                              extra={"negative_sampling": {"protocol": "fixed", "files": ["x.tsv"]}}))
        with pytest.raises(NotImplementedError, match="negative sampling"):
            run_experiment(str(p))
    finally:
        convneumf.ConvNeuMF.train = orig
    assert not trained
