"""NonNegMF on the GPU: each kernel against the oracle bit for bit (dots, est, the biases, the row updates with a zero
denominator, the bias chain in global memory), the model against the reference's goldens after every epoch, its
scores and lists, reruns, the weights round trip, and the reference's run_experiment on the NonNegMF block at C1
scale."""
import os

import numpy as np
import pytest
import torch

import c1_harness as c1h
from c1_harness import DEV, GOLD, dev_csr, to_dev
from oracle import nonneg_mf as onm
from oracle.slope_one import isolated
from elliot_b200 import ops

pytestmark = pytest.mark.gpu
_G = dict(np.load(os.path.join(GOLD, "nonneg_mf_cases.npz")))
CASES = list(_G["cases"])
EPOCHS = int(_G["epochs"])


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(a, b):
    """Bit-equal fp64 arrays, except that any NaN matches any NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(_bits(np.where(na, 0.0, a)), _bits(np.where(nb, 0.0, b)))


def _case(name):
    U, I, F = (int(x) for x in _G[f"{name}_shape"])
    return dict(U=U, I=I, F=F, indptr=_G[f"{name}_indptr"], items=_G[f"{name}_items"].astype(np.int64),
                vals=_G[f"{name}_ratings"], mu=float(_G[f"{name}_mu"]), lr=float(_G[f"{name}_lr"]),
                reg=float(_G[f"{name}_reg"]), seed=int(_G[f"{name}_seed"]))


class _Data:
    """The DataSet fields NonNegMFModel reads: i_train_dict in the given dict order."""

    def __init__(self, indptr, items, vals, n_items):
        U = len(indptr) - 1
        self.users, self.items = list(range(U)), list(range(n_items))
        self.i_train_dict = {u: {int(i): float(v) for i, v in zip(items[indptr[u]:indptr[u + 1]], vals[indptr[u]:indptr[u + 1]])}
                             for u in range(U)}


def _csc(indptr, items, n_items):
    pos = np.argsort(items, kind="stable")
    c_indptr = np.concatenate([[0], np.cumsum(np.bincount(items, minlength=n_items))]).astype(np.int64)
    return c_indptr, onm.row_of(indptr)[pos], pos


def _mask(c):
    R = np.zeros((c["U"], c["I"]), bool)
    R[onm.row_of(c["indptr"]), c["items"]] = True
    return dev_csr(R)[:2]


# ---------------------------------------------------------------- 1. the kernels against the oracle
def _epoch_kernels(P, Q, bu, bi, c):
    """One epoch through the three entry points; returns host (dots, est, bu, bi, P, Q)."""
    ip, it, r = to_dev(c["indptr"]), to_dev(c["items"], torch.int32), to_dev(c["vals"])
    Pd, Qd, bud, bid = to_dev(P), to_dev(Q), to_dev(bu), to_dev(bi)
    d = ops.nnmf_dots_f64(Pd, Qd, ip, it)
    est = ops.nnmf_bias_chain_f64(ip, it, r, d, c["mu"], c["lr"], c["reg"], bud, bid)
    ci, cu, cp = _csc(c["indptr"], c["items"], c["I"])
    Qn = ops.nnmf_row_update_f64(to_dev(ci), to_dev(cu, torch.int32), to_dev(cp), r, est, Pd, Qd, c["reg"])
    Pn = ops.nnmf_row_update_f64(ip, it, None, r, est, Qd, Pd, c["reg"])
    return [x.cpu().numpy() for x in (d, est, bud, bid, Pn, Qn)]


@pytest.mark.parametrize("name", CASES)
def test_kernels_match_the_oracle_every_epoch(name):
    c = _case(name)
    P, Q = _G[f"{name}_P"][0], _G[f"{name}_Q"][0]
    bu, bi = np.zeros(c["U"]), np.zeros(c["I"])
    for e in range(EPOCHS):
        d, est, gbu, gbi, gP, gQ = _epoch_kernels(P, Q, bu, bi, c)
        P, Q, od, oest = onm.epoch(P, Q, bu, bi, c["mu"], c["indptr"], c["items"], c["vals"], c["lr"], c["reg"])
        for key, got, want in (("dot", d, od), ("est", est, oest), ("bu", gbu, bu), ("bi", gbi, bi), ("P", gP, P),
                               ("Q", gQ, Q)):
            assert np.array_equal(_bits(got), _bits(want)), (name, e, key)
        assert np.array_equal(_bits(P), _bits(_G[f"{name}_P"][e + 1])), (name, e)


def test_row_update_reproduces_zero_denominators():
    g = np.random.default_rng(11)
    F, n_rows, n_cols = 6, 5, 9
    counts = np.array([3, 0, 4, 2, 5])
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    cols = g.integers(0, n_cols, counts.sum())
    pos = g.permutation(counts.sum())
    r = g.integers(0, 6, counts.sum()).astype(np.float64)
    est = g.normal(size=counts.sum())
    T, S = g.normal(size=(n_cols, F)), g.normal(size=(n_rows, F))
    est[pos[indptr[2]:indptr[3]]] = 0.0                 # row 2: den = 0 + (n reg) S = 0 where S = 0: 0 * inf or NaN
    S[2, :3] = 0.0
    for reg in (0.1, 0.0):
        want = onm.row_update(S, T, np.repeat(np.arange(n_rows), counts), cols, counts, r[pos], est[pos], reg)
        got = ops.nnmf_row_update_f64(to_dev(indptr), to_dev(cols, torch.int32), to_dev(pos), to_dev(r), to_dev(est),
                                      to_dev(T), to_dev(S), reg).cpu().numpy()
        assert _same(got, want), reg
        assert np.isnan(got[1]).all()                   # a row without entries: 0 / 0
        assert not np.isfinite(got[2, :3]).any()
    est[pos[indptr[4]:indptr[5]]] = 0.0
    S[4] = 1.5
    want = onm.row_update(S, T, np.repeat(np.arange(n_rows), counts), cols, counts, r[pos], est[pos], 0.0)
    Sd = to_dev(S)
    got = ops.nnmf_row_update_f64(to_dev(indptr), to_dev(cols, torch.int32), to_dev(pos), to_dev(r), to_dev(est),
                                  to_dev(T), Sd, 0.0, out=Sd).cpu().numpy()             # in place
    assert _same(got, want)
    assert np.isinf(got[4]).any()                       # num / +-0 -> +-inf times a non-zero S


def test_bias_chain_in_global_memory():
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    I = optin // 8 + 1000                               # bi does not fit the opt-in shared memory
    g = np.random.default_rng(5)
    U = 400
    counts = g.integers(1, 60, U)
    counts[3] = 0                                       # a user without ratings keeps its bias
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    hot = g.choice(I, 80, replace=False)                # items many users share: long dependency runs through bi
    items = np.concatenate([g.choice(hot if u % 2 else I, c, replace=False) for u, c in enumerate(counts)])
    vals = g.integers(0, 6, items.size).astype(np.float64)
    d = g.normal(size=items.size) * 3
    bu0, bi0 = g.normal(size=U), g.normal(size=I)
    bu, bi = bu0.copy(), bi0.copy()
    oest = onm.bias_chain(bu, bi, 3.25, indptr, items, vals, d, 0.01, 0.07)
    bud, bid = to_dev(bu0), to_dev(bi0)
    est = ops.nnmf_bias_chain_f64(to_dev(indptr), to_dev(items, torch.int32), to_dev(vals), to_dev(d), 3.25, 0.01, 0.07,
                                  bud, bid)
    assert np.array_equal(_bits(est.cpu().numpy()), _bits(oest))
    assert np.array_equal(_bits(bud.cpu().numpy()), _bits(bu)) and np.array_equal(_bits(bid.cpu().numpy()), _bits(bi))
    assert bud[3].item() == bu0[3]


# ---------------------------------------------------------------- 2. the model against the reference's goldens
def _model(c):
    from elliot_b200.recommender.nonneg_mf import NonNegMFModel
    return NonNegMFModel(_Data(c["indptr"], c["items"], c["vals"], c["I"]), c["U"], c["I"], np.float32(c["mu"]), c["F"],
                         c["reg"], c["lr"], random_seed=c["seed"], device=DEV)


@pytest.mark.parametrize("name", CASES)
def test_model_matches_the_reference_every_epoch(name):
    c = _case(name)
    m = _model(c)
    for e in range(EPOCHS + 1):
        if e:
            m.train_step()
        s = m.get_model_state()
        for key, ref in (("_user_embeddings", "P"), ("_item_embeddings", "Q"), ("_user_bias", "bu"), ("_item_bias", "bi")):
            assert np.array_equal(_bits(s[key]), _bits(_G[f"{name}_{ref}"][e])), (name, e, key)
    K = int(_G["topk"])
    idx, val = (x.cpu().numpy() for x in m.topk(K + 1, *_mask(c)))
    ti, tv = _G[f"{name}_topk_idx"], _G[f"{name}_topk_val"]
    assert np.array_equal(idx[:, :K] >= 0, ti >= 0)
    # the reference's ddot differs from the kernel's sum in the last bits only
    P, Q, bu, bi = (_G[f"{name}_{k}"][-1] for k in ("P", "Q", "bu", "bi"))
    scale = np.abs(P) @ np.abs(Q).T + np.abs(bi)[None, :] + np.abs(bu)[:, None] + abs(c["mu"])
    ok = ti >= 0
    rows = np.nonzero(ok)[0]
    mine = onm.scores(P, Q, bu, bi, c["mu"])
    assert np.all(np.abs(mine[rows, ti[ok]] - tv[ok]) <= 1e-12 * scale[rows, ti[ok]])
    got = np.where(idx[:, :K] >= 0, val[:, :K], -np.inf)
    assert np.all(np.abs(got[ok] - tv[ok]) <= 1e-12 * scale[rows, ti[ok]])
    iso = isolated(val, margin=2e-12 * scale.max())[:, :K]
    assert np.array_equal(idx[:, :K][iso], ti[iso]), name
    assert iso.sum() > 0.8 * ok.sum()


def test_rerun_and_weights_round_trip(tmp_path):
    c = _case("stars")
    a, b = _model(c), _model(c)
    for _ in range(2):
        a.train_step()
        b.train_step()
    mask = _mask(c)
    (ia, va), (ib, vb) = a.topk(20, *mask), b.topk(20, *mask)
    assert torch.equal(ia, ib) and torch.equal(va.view(torch.int64), vb.view(torch.int64))
    for x, y in ((a.P, b.P), (a.Q, b.Q), (a.bu, b.bu), (a.bi, b.bi)):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
    a.save_weights(str(tmp_path / "w"))
    d = _model(c)
    d.load_weights(str(tmp_path / "w"))
    idd, vd = d.topk(20, *mask)
    assert torch.equal(ia, idd) and torch.equal(va.view(torch.int64), vd.view(torch.int64))
    a.train_step()
    d.train_step()                                      # training goes on from the restored tables
    assert torch.equal(a.P.view(torch.int64), d.P.view(torch.int64))


# ---------------------------------------------------------------- 3. run_experiment at C1 scale
c1 = c1h.c1_fixture("nonneg_mf_c1.npz")


@pytest.mark.parametrize("ev", ["host", "device"])
def test_run_experiment_matches_the_reference_run(c1, ev):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / f"NonNegMF_{ev}"
    res = c1h.run(out, synth_c1.nonneg_mf_yaml(tsv, str(out), model_extra=f"      b200_eval: {ev}\n"), ev == "device")
    c1h.assert_metrics(res, g["metrics"].tolist(), g["test_metrics"], "NonNegMF", ev)
    if ev == "device":
        c1h.assert_no_rec_files(out)
        return
    files = sorted(os.listdir(out / "recs"))
    assert files == sorted(g["rec_files"].tolist()), files
    rec = np.loadtxt(out / "recs" / str(g["rec_file"]), delimiter="\t")
    users = np.unique(g["rec_users"])
    mine = rec[np.isin(rec[:, 0].astype(np.int64), users)]
    gu, gi, gs = g["rec_users"], g["rec_items"], g["rec_scores"]
    assert np.array_equal(np.unique(mine[:, 0]).astype(np.int64), users)
    same = total = 0
    for u in users:
        a, b = mine[mine[:, 0] == u], (gu == u)
        assert len(a) == b.sum() == 10
        assert np.all(np.abs(a[:, 2] - gs[b]) <= 1e-9 * np.abs(gs[b]).max()), u
        iso = isolated(gs[b][None, :], margin=1e-9 * np.abs(gs[b]).max())[0]
        iso[-1] = False                                 # the k+1-th value is not in the file
        assert np.array_equal(a[iso, 1].astype(np.int64), gi[b][iso]), u
        same += iso.sum()
        total += 10
    assert same > 0.5 * total, (same, total)


def test_restore_evaluates_the_saved_tables(c1):
    from elliot_b200 import synth_c1
    g, d, tsv = c1
    out = d / "NonNegMF_saved"
    block = "      epochs: 2\n      factors: 10\n      lr: 0.001\n      reg: 0.1\n"
    first = c1h.run(out, synth_c1.experiment_yaml(tsv, str(out), "NonNegMF", block, meta=("save_weights: True",)))
    again = c1h.run(out, synth_c1.experiment_yaml(tsv, str(out), "NonNegMF", block, meta=("restore: True",)))
    assert again["test_results"] == first["test_results"]
