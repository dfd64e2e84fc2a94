"""GPU tests of UserAutoRec / ItemAutoRec (csrc/autorec.cu, recommender/autorec.py): the whole training step against the
fp64 restatement of oracle/autorec.py at bounds derived from the fp32 unit roundoff, H and the row lengths (long rows
split over many CTAs included), the determinism of dpre1 and the loss, one Keras Adam step, both models' top-k and
AUC / GAUC rank pass, C1 runs through run_experiment, and the refusals."""
import pickle
import random

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import yaml

from elliot_b200 import synth_c1
from elliot_b200.recommender import autorec as model_mod
from elliot_b200.recommender.autorec import LINEAR, SIGMOID, AutoRecModel
from oracle import autorec as oracle
from oracle import tf_models as tfm
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 2.0 ** -24
ACTS = {"linear": LINEAR, "sigmoid": SIGMOID}


def _dev(a, dt=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)


def _csr(X):
    m = sp.csr_matrix(X.astype(np.float32)); m.sort_indices()
    return _dev(m.indptr.astype(np.int64)), _dev(m.indices.astype(np.int32)), _dev(m.data.astype(np.float32))


def _model(X, H, act, lr=1e-3, seed=5):
    n = X.shape[1]
    return AutoRecModel(n, n, H, lr, ACTS[act], seed, DEV, _csr(X))


def _host(m):
    W1, b1, W2t, b2 = (t.double().cpu().numpy() for t in m.P)
    return W1, b1, W2t, b2[:m.n_out]


def _h_bound(X, W1, b1):
    """The encoder on the device: z is a sum of n_b + 1 fp32 terms (the row's W1 rows and b1), then __expf (error
    2 + 1.173 |z| ulp) and a division.  |dh| <= h (1 - h) (dz + (4 + 2.4 |z|) u) + 3 u h."""
    z = X @ W1 + b1
    h = oracle.sigmoid(z)
    dz = ((X != 0).sum(1, keepdims=True) + 2) * U32 * (X @ np.abs(W1) + np.abs(b1))
    return h, h * (1 - h) * (dz + (4 + 2.4 * np.abs(z)) * U32) + 3 * U32 * h


def _step_bounds(X, h, W2t, b2, act):
    """Bounds of the device's decoder step given its own h (fp64 copy), from the fp32 unit roundoff u:
    o = h . W2[i] + b2[i] is an H-term fp32 dot plus a bias, |do| <= (H + 2) u (|h| . |W2[i]| + |b2[i]|);
    sigmoid (expf, 2 ulp; a sum and a division): |dr| <= r (1 - r) (do + 4 u) + 3 u r; e = 1 - r: |de| <= dr + u |e|;
    g = -2 e act' / B: |dg| <= 2 / B (de act' + |e| d(act')) + 4 u |g| with d(act') <= dr + 3 u act';
    dW2[i] and db2[i] add c_i fp32 products by reductions (c_i the batch rows holding i), dh_b adds n_b products (n_b the
    row's entries), dpre1 = dh h (1 - h) three more roundings, dW1 and db1 sums of c_j and B of those."""
    B, H = X.shape[0], h.shape[1]
    M = X != 0
    o = h @ W2t.T + b2
    do = (H + 2) * U32 * (np.abs(h) @ np.abs(W2t).T + np.abs(b2))
    if act == "sigmoid":
        r = oracle.sigmoid(o)
        dr = r * (1 - r) * (do + 4 * U32) + 3 * U32 * r
        ap = r * (1 - r)
        dap = dr + 3 * U32 * ap
    else:
        r, dr, ap, dap = o, do, np.ones_like(o), np.zeros_like(o)
    e = np.where(M, X - r, 0.0)
    de = np.where(M, dr + U32 * np.abs(e), 0.0)
    g = -2.0 * e * ap / B
    dg = np.where(M, 2.0 / B * (de * ap + np.abs(e) * dap) + 4 * U32 * np.abs(g), 0.0)
    c = M.sum(0)
    nb = M.sum(1, keepdims=True)
    b = {"loss": (2 * np.abs(e) * de + de * de).sum() / B + 1e-14 * (e * e).sum() / B,
         "dW2": (np.abs(h).T @ dg + (np.abs(h).T @ np.abs(g)) * (c + 2) * U32).T,          # [n_out][H] as the device
         "db2": dg.sum(0) + (c + 2) * U32 * np.abs(g).sum(0)}
    dh = g @ W2t
    ddh = dg @ np.abs(W2t) + (nb + 2) * U32 * (np.abs(g) @ np.abs(W2t))
    sh = h * (1 - h)
    ddp = ddh * sh + 3 * U32 * np.abs(dh) * sh
    dp = np.abs(dh * sh)
    b["dpre1"] = ddp
    b["dW1"] = np.abs(X).T @ ddp + (c[:, None] + 2) * U32 * (np.abs(X).T @ dp)
    b["db1"] = ddp.sum(0) + (B + 2) * U32 * dp.sum(0)
    return b


def _run_step(m, rows):
    m._loss.zero_()
    h, dpre1 = m.grads(_dev(rows.astype(np.int32)))
    torch.cuda.synchronize()
    got = {"loss": m._loss.item(), "h": h.double().cpu().numpy(), "dpre1": dpre1.double().cpu().numpy(),
           "dW1": m.G[0].double().cpu().numpy(), "db1": m.G[1].double().cpu().numpy(),
           "dW2": m.G[2].double().cpu().numpy(), "db2": m.G[3].double().cpu().numpy()[:m.n_out]}
    for gr in m.G:
        gr.zero_()
    return got


def _check_step(X_all, rows, H, act):
    m = _model(X_all, H, act)
    W1, b1, W2t, b2 = _host(m)
    got = _run_step(m, rows)
    X = X_all[rows]
    h64, dh = _h_bound(X, W1, b1)
    assert (np.abs(got["h"] - h64) <= dh).all()
    # the whole step restated on the device's own encoder output (the decoder's input)
    loss, dW1, db1, dW2, db2 = oracle.step(X, W1, b1, W2t.T, b2, act, h=got["h"])
    bd = _step_bounds(X, got["h"], W2t, b2, act)
    assert abs(got["loss"] - loss) <= bd["loss"], (got["loss"], loss, bd["loss"])
    for key, want in (("dW1", dW1), ("db1", db1), ("dW2", dW2.T), ("db2", db2)):
        err = np.abs(got[key] - want)
        assert (err <= bd[key] + 1e-30).all(), (key, (err / (bd[key] + 1e-30)).max())
    # inputs and outputs no batch row holds get exactly 0
    untouched = X.sum(0) == 0
    assert untouched.any() or X.shape[0] >= 64
    assert not got["dW2"][untouched].any() and not got["db2"][untouched].any() and not got["dW1"][untouched].any()
    empty = X.sum(1) == 0
    assert not got["dpre1"][empty].any()
    return m, got


def _matrix(rs, n_rows, n_cols, density):
    X = (rs.rand(n_rows, n_cols) < density).astype(np.float64)
    X[3] = 0.0                                                           # an empty row
    return X


@pytest.mark.parametrize("act", ["linear", "sigmoid"])
@pytest.mark.parametrize("H", [4, 64, 500, 1024])
@pytest.mark.parametrize("B", [1, 7, 512])
def test_step_matches_fp64(act, H, B):
    rs = np.random.RandomState(H + B)
    X = _matrix(rs, 600, 300, 0.2)
    rows = rs.permutation(600)[:B]
    if B > 1:
        rows[1] = 3                                                      # the empty row is in the batch
    _check_step(X, rows, H, act)


@pytest.mark.parametrize("act", ["linear", "sigmoid"])
@pytest.mark.parametrize("H", [64, 500])
def test_step_long_row_split_over_ctas(act, H):
    """A row of 51 000 entries spans 100-200 segments of the persistent grid; its dh segments are combined in order."""
    rs = np.random.RandomState(H)
    n = 52_000
    X = np.zeros((8, n))
    X[0, rs.choice(n, 51_000, replace=False)] = 1.0
    X[1, rs.choice(n, 300, replace=False)] = 1.0
    X[2, rs.choice(n, 5, replace=False)] = 1.0
    _check_step(X, np.array([0, 3, 2, 1]), H, act)


@pytest.mark.parametrize("H", [64, 500])
def test_dpre1_and_loss_are_deterministic(H):
    rs = np.random.RandomState(1)
    X = _matrix(rs, 600, 20_000, 0.02)
    X[5, :] = (rs.rand(20_000) < 0.9)                                   # a row of ~18 000 entries: many segments
    rows = np.r_[5, rs.permutation(np.delete(np.arange(600), 5))[:511]]
    m = _model(X, H, "sigmoid")
    a, b = _run_step(m, rows), _run_step(m, rows)
    assert a["loss"] == b["loss"]
    assert np.array_equal(a["dpre1"], b["dpre1"])


def test_adam_step_matches_keras():
    rs = np.random.RandomState(4)
    X = _matrix(rs, 300, 200, 0.1)
    m = _model(X, 64, "sigmoid", lr=0.01)
    opt = tfm.KerasAdam(0.01)
    T = [p.double().cpu().numpy() for p in m.P]
    for step in range(2):
        m.grads(_dev(rs.permutation(300)[:128].astype(np.int32)))
        G = [gr.double().cpu().numpy() for gr in m.G]
        m.adam()
        opt.begin_step()
        for k, (p, gr) in enumerate(zip(m.P, G)):
            opt.apply(k, T[k], gr)
            got = p.double().cpu().numpy()
            assert np.abs(got - T[k]).max() <= 8 * U32 * (np.abs(T[k]).max() + 0.01), (step, k)
            T[k] = got
        assert all(not gr.any() for gr in m.G)


# ---------------------------------------------------------------- scoring
def _mask_of(X):
    m = sp.csr_matrix(X); m.sort_indices()
    return m.indptr.astype(np.int64), m.indices.astype(np.int32)


@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("H", [64, 500])
def test_user_topk_matches_fp64(k, H):
    rs = np.random.RandomState(k + H)
    X = _matrix(rs, 400, 700, 0.05)
    m = _model(X, H, "linear")
    for p in m.P[2:]:
        p.mul_(3.0)                                                      # spread the scores
    ip, ix = _mask_of(X)
    idx, val = m.topk(k, _dev(ip), _dev(ix))
    h = m.hidden().double().cpu().numpy()
    W1, b1, W2t, b2 = _host(m)
    h64, dh = _h_bound(X, W1, b1)
    assert (np.abs(h - h64) <= dh).all()
    f, t = check_topk_fp64(h, W2t, b2, H, k, ip, ix, np.arange(400), idx.cpu().numpy(), val.cpu().numpy(), U32)
    assert t > 0 and f > t // 2


def _item_lists_check(idx, val, S, dS, mask, k):
    """Device lists (ids, sigmoid values) against the literal fp64 scores S [U][I] (column j = item j under perm) with
    per-score bounds dS: values within the bound of their item's fp64 score, the returned set's sorted scores within twice
    the bound of the literal top k, and ids equal wherever the literal score is isolated by more than twice the bound
    (inside runs of equal fp32 scores, where the sigmoid saturates, the order is the logit's, not the index's)."""
    Sm = np.where(mask, S, -np.inf)
    want_v, want_i = oracle.top_k(S, mask, k + 1)
    iso = checked = 0
    for u in range(S.shape[0]):
        got = idx[u] >= 0
        assert got.sum() == np.isfinite(want_v[u, :k]).sum()
        j = idx[u][got]
        assert mask[u, j].all() and len(np.unique(j)) == len(j)
        bd = dS[u].max()
        assert (np.abs(val[u][got] - Sm[u, j]) <= dS[u, j]).all(), u
        assert (np.abs(np.sort(Sm[u, j])[::-1] - want_v[u, :got.sum()]) <= 2 * bd).all(), u
        gaps = np.diff(-want_v[u])
        sep = ~np.isfinite(gaps) | (gaps > 2 * bd)
        ok = sep & np.r_[True, sep[:-1]]
        for r in np.flatnonzero(ok[:got.sum()]):
            checked += 1
            iso += idx[u, r] == want_i[u, r]
    assert checked > 0 and iso == checked


def _item_scores(XT, W1, b1, W2t, b2, perm, H):
    """The literal restatement's scores [U][I] and their bounds: V = the encoder (bound _h_bound), the logit an H-term fp32
    dot of the device's operands, |dlogit| <= (H + 2) u |W2| . |V| + |W2| . dV; then the bias, the sigmoid (__expf) and
    its division: |ds| <= s (1 - s) (dlogit + (5 + 2.4 |l|) u) + 3 u s."""
    V, dV = _h_bound(XT[perm], W1, b1)
    L = W2t @ V.T + b2[:, None]
    dL = (H + 2) * U32 * (np.abs(W2t) @ np.abs(V).T + np.abs(b2)[:, None]) + np.abs(W2t) @ dV.T
    S = oracle.sigmoid(L)
    return S, S * (1 - S) * (dL + (5 + 2.4 * np.abs(L)) * U32) + 3 * U32 * S


@pytest.mark.parametrize("k", [10, 50])
@pytest.mark.parametrize("H", [64, 500])
def test_item_topk_matches_literal_under_permutation(k, H):
    rs = np.random.RandomState(k + H)
    X = _matrix(rs, 500, 300, 0.05)                                      # 500 users x 300 items
    XT = X.T.copy()
    m = _model(XT, H, "sigmoid")
    perm = rs.permutation(300)
    ip, ix = _mask_of(X)
    idx, val = (t.cpu().numpy() for t in m.item_topk(perm.tolist(), k, _dev(ip), _dev(ix)))
    W1, b1, W2t, b2 = _host(m)
    lit_v, lit_i = oracle.get_recommendations_item(XT, W1, b1, W2t.T, b2, perm, X == 0, k)
    S, dS = _item_scores(XT, W1, b1, W2t, b2, perm, H)
    assert np.allclose(np.take_along_axis(S, lit_i, 1), lit_v, rtol=1e-12)
    _item_lists_check(idx, val.astype(np.float64), S, dS, X == 0, k)


def _rel(rs, X, n_max=12):
    free = [np.flatnonzero(X[u] == 0) for u in range(X.shape[0])]
    rel = [np.sort(rs.choice(c, size=min(rs.randint(0, n_max), len(c)), replace=False)) for c in free]
    return rel, np.r_[0, np.cumsum([len(r) for r in rel])].astype(np.int64), np.concatenate(rel).astype(np.int32)


def _check_counts(n_pos, sum_c, Ssc, bound, X, rel):
    """The rank pass counts against the fp64 scores of the device's operands: every relevant item counted, and the non-relevant
    items ahead between those surely ahead and those possibly ahead (within the fp32 dot products' rounding)."""
    for u in range(X.shape[0]):
        s = np.where(X[u] == 0, Ssc[u], -np.inf)
        other = np.isfinite(s)
        other[rel[u]] = False
        lo = sum(int((s[other] > s[r] + bound[u, r] + bound[u, other]).sum()) for r in rel[u])
        hi = sum(int((s[other] >= s[r] - bound[u, r] - bound[u, other]).sum()) for r in rel[u])
        assert n_pos[u] == len(rel[u]) and lo <= sum_c[u] <= hi, u
    assert n_pos.sum() > 0 and sum_c.sum() > 0


def test_user_rank_pass_gives_fp64_counts():
    rs = np.random.RandomState(9)
    X = _matrix(rs, 200, 300, 0.05)
    m = _model(X, 64, "linear")
    m.P[2].mul_(3.0)
    rel, rp, ri = _rel(rs, X)
    ip, ix = _mask_of(X)
    n_pos, sum_c = (t.cpu().numpy() for t in m.rank(_dev(rp), _dev(ri), _dev(ip), _dev(ix)))
    h = m.hidden().double().cpu().numpy()
    _, _, W2t, b2 = _host(m)
    bound = 66 * U32 * (np.abs(h) @ np.abs(W2t).T + np.abs(b2))
    _check_counts(n_pos, sum_c, h @ W2t.T + b2, bound, X, rel)


def test_item_rank_pass_gives_fp64_counts():
    rs = np.random.RandomState(10)
    X = _matrix(rs, 200, 300, 0.05)
    XT = X.T.copy()
    m = _model(XT, 64, "sigmoid")
    perm = rs.permutation(300)
    rel, rp, ri = _rel(rs, X)
    ip, ix = _mask_of(X)
    n_pos, sum_c = (t.cpu().numpy() for t in m.item_rank(perm.tolist(), _dev(rp), _dev(ri), _dev(ip), _dev(ix)))
    V = m.item_operand(perm.tolist()).double().cpu().numpy()
    _, _, W2t, _ = _host(m)
    bound = 66 * U32 * (np.abs(W2t) @ np.abs(V).T)
    _check_counts(n_pos, sum_c, W2t @ V.T, bound, X, rel)


# ---------------------------------------------------------------- C1 runs through run_experiment
@pytest.fixture(scope="module")
def c1_tsv(tmp_path_factory):
    tsv = str(tmp_path_factory.mktemp("autorec_c1") / "dataset.tsv")
    synth_c1.write_tsv(tsv)
    return tsv


def _c1_yaml(tsv, out, key, block, meta, metrics=("nDCG", "AUC"), extra=None):
    cfg = yaml.safe_load(synth_c1.experiment_yaml(tsv, out, key, "", metrics=metrics, meta=()))
    cfg["experiment"]["models"][key] = dict(block, meta=meta)
    if extra:
        cfg["experiment"].update(extra)
    return yaml.safe_dump(cfg)


class _Recorder:
    """Records, through the model code, the rows of every train step, the permutation of every ItemAutoRec list and rank
    pass, the random state around each rank pass, every list, and the models built."""

    def __init__(self):
        self.rows, self.list_perms, self.rank_perms, self.rank_states, self.lists, self.models = [], [], [], [], [], []
        M, R = AutoRecModel, model_mod._AutoRec
        self.orig = [(M, "train_step"), (M, "item_topk"), (M, "item_rank"), (M, "topk"), (R, "train"),
                     (model_mod.ItemAutoRec, "get_rank_tensors")]
        self.saved = [getattr(c, n) for c, n in self.orig]
        step, item_topk, item_rank, topk, train, grt = self.saved
        rec = self

        def w_step(self_, rows):
            rec.rows.append(rows.cpu().numpy())
            return step(self_, rows)

        def w_item_topk(self_, perm, *a):
            rec.list_perms.append(list(perm))
            out = item_topk(self_, perm, *a)
            rec.lists.append(tuple(t.cpu().numpy() for t in out))
            return out

        def w_item_rank(self_, perm, *a):
            rec.rank_perms.append(list(perm))
            return item_rank(self_, perm, *a)

        def w_topk(self_, *a):
            out = topk(self_, *a)
            rec.lists.append(tuple(t.cpu().numpy() for t in out))
            return out

        def w_train(self_):
            rec.models.append(self_)
            return train(self_)

        def w_grt(self_, *a):
            before = random.getstate()
            out = grt(self_, *a)
            rec.rank_states.append(before == random.getstate())
            return out
        for (c, n), f in zip(self.orig, (w_step, w_item_topk, w_item_rank, w_topk, w_train, w_grt)):
            setattr(c, n, f)

    def restore(self):
        for (c, n), f in zip(self.orig, self.saved):
            setattr(c, n, f)


def _metrics(result):
    """nDCG and AUC at 10 on the test split from one evaluate() result."""
    r = result[10]["test_results"]
    return {k: r[k] for k in ("nDCG", "AUC")}


@pytest.mark.parametrize("key", ["UserAutoRec", "ItemAutoRec"])
@pytest.mark.parametrize("batch", [512, -1])
def test_c1_run_trains_replays_evaluates_saves_and_restores(c1_tsv, tmp_path, key, batch):
    from elliot_b200 import run_experiment
    epochs = 3
    block = {"epochs": epochs, "batch_size": batch, "lr": 0.001, "seed": 7}
    rec = _Recorder()
    try:
        p = tmp_path / "cfg.yml"
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, block, {"save_weights": True, "save_recs": False}))
        res = run_experiment(str(p))[0]
        m = rec.models[-1]
        n_train_rows = len(rec.rows)
        # device metrics against the host path on the same model state (ItemAutoRec: under the same draw)
        st = random.getstate()
        m._params.b200_eval = "device"
        m.evaluate()
        dev = _metrics(m._results[-1])
        random.setstate(st)
        m._params.b200_eval = "host"
        m.evaluate()
        host = _metrics(m._results[-1])
        random.setstate(st)
        # the same lists; the two evaluators may sum a metric in different orders
        assert all(np.isfinite(v) and dev[k] == pytest.approx(v, rel=1e-12) for k, v in host.items()), (dev, host)
        saved = pickle.load(open(m._saving_filepath, "rb"))
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, block, {"restore": True, "save_recs": False}))
        n_before = len(rec.list_perms)
        again = run_experiment(str(p))[0]
        restored = rec.models[-1]
    finally:
        rec.restore()
    item = key == "ItemAutoRec"
    assert res["name"].startswith(key + "_") and len(res["history"]) == epochs
    assert len(rec.rows) == n_train_rows                                 # the restore run trains no step
    n_rows = m._num_items if item else m._num_users
    B = m._data.transactions if batch < 1 else batch
    assert m._batch_size == B
    per_epoch = -(-n_rows // B)
    assert n_train_rows == epochs * per_epoch
    draws = oracle.replay(n_rows, m._num_items, epochs, item)
    orders = [d for d in draws if d[0] == "epoch"]
    for e in range(epochs):
        got = np.concatenate(rec.rows[e * per_epoch:(e + 1) * per_epoch])
        assert got.tolist() == orders[e][2], e
    if item:
        evals = [d[2] for d in draws if d[0] == "eval"]
        assert rec.list_perms[:epochs] == evals                          # one draw per evaluation, where the reference draws
        assert rec.rank_perms[:epochs] == evals and all(rec.rank_states)
        assert rec.list_perms[n_before:] == [oracle.replay_restore(m._num_items)]
    # the loss falls over the epochs (evaluate() gets the epoch sum / (epoch + 1))
    sums = [l * (e + 1) for e, l in enumerate(m._losses[:epochs])]
    assert np.isfinite(sums).all() and sums[-1] < sums[0], sums
    # the restored model's lists are those the restatement predicts from the saved weights
    assert all(np.array_equal(a, b) for a, b in zip(saved["P"], (t.cpu().numpy() for t in restored._model.P)))
    idx, val = rec.lists[-1]
    X = m._data.sp_i_train.toarray().astype(np.float64)
    W1, b1, W2t, b2 = (a.astype(np.float64) for a in saved["P"])
    H = W1.shape[1]
    ip, ix = (t.cpu().numpy() for t in (m._indptr, m._sorted_idx))
    if item:
        perm = oracle.replay_restore(m._num_items)
        S, dS = _item_scores(X.T.copy(), W1, b1, W2t, b2[:m._num_users], perm, H)
        _item_lists_check(idx, val.astype(np.float64), S, dS, X == 0, 10)
    else:
        h = restored._model.hidden().double().cpu().numpy()
        h64, dh = _h_bound(X, W1, b1)
        assert (np.abs(h - h64) <= dh).all()
        f, t = check_topk_fp64(h, W2t, b2[:m._num_items], H, 10, ip, ix, np.arange(m._num_users), idx, val, U32)
        assert t > 0 and f > t // 2
    assert np.isfinite(again["test_results"][10]["nDCG"])


@pytest.mark.parametrize("key", ["UserAutoRec", "external.ItemAutoRec"])
def test_c1_refusals_before_training(c1_tsv, tmp_path, key):
    import os
    from elliot_b200 import run_experiment
    rec = _Recorder()
    extra = {"external_models_path": os.path.join(os.path.dirname(synth_c1.__file__), "plugin.py")} if "." in key else {}
    try:
        p = tmp_path / "cfg.yml"
        for block, metrics, err, match in (({"epochs": 1, "hidden_neuron": 30}, ("nDCG",), ValueError, "multiple of 4"),
                                           ({"epochs": 1, "hidden_neuron": 2048}, ("nDCG",), ValueError, "multiple of 4"),
                                           ({"epochs": 1}, ("nDCG", "MAE"), Exception, "cannot evaluate MAE")):
            p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, block, {"save_recs": False}, metrics=metrics, extra=extra))
            with pytest.raises(err, match=match):
                run_experiment(str(p))
        p.write_text(_c1_yaml(c1_tsv, str(tmp_path), key, {"epochs": 1}, {"save_recs": False},
                              extra=dict(extra, negative_sampling={"protocol": "fixed", "files": ["x.tsv"]})))
        with pytest.raises(NotImplementedError):
            run_experiment(str(p))
    finally:
        rec.restore()
    assert rec.rows == []
