"""NeuMF kernels + tensor-core MLP vs the fp64 numpy restatement (TensorFlow parity UNPINNED)."""
import numpy as np
import pytest
import torch

from elliot_b200 import ops
from elliot_b200.recommender.neumf import NeuralMatrixFactorizationModel
from oracle import tf_models as tfm

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ref_params(m):
    f = m.f
    g = lambda k: m.P[k].double().cpu().numpy()
    return {"U_mf": g("U_mf"), "I_mf": g("I_mf"), "U_mlp": g("U_mlp"), "I_mlp": g("I_mlp"),
            "W1": g("W1").T, "b1": g("b1")[:4 * f], "W2": g("W2").T, "b2": g("b2")[:2 * f], "W3": g("W3").T, "b3": g("b3")[:f],
            "wp": g("wp"), "bp": float(g("bp")[0])}


def test_train_step_matches_restatement():
    nu, ni, f, B = 120, 90, 16, 700
    m = NeuralMatrixFactorizationModel(nu, ni, f, 1e-3, 42, DEV)
    for k in ("b1", "b2", "b3", "bp"):
        m.P[k].normal_(0, 0.05)
    for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
        m.P[k].mul_(4.0)                                     # larger activations -> meaningful ReLU pattern
    P = _ref_params(m)
    rs = np.random.RandomState(0)
    u = rs.randint(0, nu, B).astype(np.int32); i = rs.randint(0, ni, B).astype(np.int32)
    y = (rs.rand(B) < 0.3).astype(np.float32)
    loss_ref, G, p_ref = tfm.neumf_forward_backward(P, u, i, y.astype(np.float64))
    loss = m.train_step((torch.from_numpy(u).to(DEV), torch.from_numpy(i).to(DEV), torch.from_numpy(y).to(DEV))).item()
    assert abs(loss - loss_ref) < 1e-2 * abs(loss_ref)
    rel = lambda a, b: np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12)
    M = lambda k: m.M[k].double().cpu().numpy() / 0.1         # first Adam step: m = 0.1 g
    # bf16 operands: rounding flips a few ReLU masks near zero, the error grows with depth (W1 is 3 layers down)
    for k, tol in (("W3", 5e-2), ("W2", 6e-2), ("W1", 1e-1)):
        assert rel(M(k), G[k].T) < tol, (k, rel(M(k), G[k].T))
    for k, n, tol in (("b3", f, 5e-2), ("b2", 2 * f, 6e-2), ("b1", 4 * f, 1e-1)):
        assert rel(M(k)[:n], G[k]) < tol, k
    assert rel(M("wp"), G["wp"]) < 2e-2 and abs(M("bp")[0] - G["bp"]) < 2e-2 * abs(G["bp"]) + 1e-6
    for k, tol in (("U_mf", 2e-2), ("I_mf", 2e-2), ("U_mlp", 1e-1), ("I_mlp", 1e-1)):
        assert rel(M(k), G[k]) < tol, (k, rel(M(k), G[k]))


def test_get_recs_equals_pointwise_forward_and_masks():
    nu, ni, f = 70, 333, 8
    m = NeuralMatrixFactorizationModel(nu, ni, f, 1e-3, 3, DEV)
    for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
        m.P[k].mul_(5.0)
    P = _ref_params(m)
    rs = np.random.RandomState(1)
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, 30), replace=False)).astype(np.int32) for _ in range(nu)]
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    mp = torch.from_numpy(indptr).to(DEV); mi = torch.from_numpy(np.concatenate(rows)).to(DEV)
    idx, val = m.get_recs_topk(10, 40, 7, mp, mi)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    for r, uu in enumerate(range(10, 40)):
        _, _, p = tfm.neumf_forward_backward(P, np.full(ni, uu), np.arange(ni), np.zeros(ni))
        p[rows[uu]] = -np.inf
        want = np.argsort(-p, kind="stable")[:7]
        assert not set(idx[r]) & set(rows[uu].tolist())
        assert np.abs(val[r] - p[idx[r]]).max() < 2e-2                     # bf16 MLP
        assert len(set(idx[r]) & set(want)) >= 5                          # near-ties may swap under bf16


def test_get_recs_lists_are_exact_with_the_fp32_checking_gemm():
    """get_recs / get_top_k (neural_matrix_factorization_model.py:119-148) with the dense layers in fp32: the masked top-7 lists
    equal the fp64 restatement's item for item (probabilities to 1e-5) — the 5-of-7 overlap accepted above is bf16 rounding of
    near-ties, not a wiring error."""
    nu, ni, f = 70, 333, 8
    with ops.exact_gemm():
        m = NeuralMatrixFactorizationModel(nu, ni, f, 1e-3, 3, DEV)
        for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
            m.P[k].mul_(5.0)
        m._refresh()
        P = _ref_params(m)
        rs = np.random.RandomState(1)
        rows = [np.sort(rs.choice(ni, size=rs.randint(1, 30), replace=False)).astype(np.int32) for _ in range(nu)]
        indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
        mp = torch.from_numpy(indptr).to(DEV); mi = torch.from_numpy(np.concatenate(rows)).to(DEV)
        idx, val = m.get_recs_topk(10, 40, 7, mp, mi)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    for r, uu in enumerate(range(10, 40)):
        _, _, p = tfm.neumf_forward_backward(P, np.full(ni, uu), np.arange(ni), np.zeros(ni))
        p[rows[uu]] = -np.inf
        want = np.argsort(-p, kind="stable")[:7]
        gaps = np.abs(np.diff(np.sort(p[np.isfinite(p)])[::-1][:8]))
        if gaps.min() > 1e-5:                                              # skip rows whose top-8 holds an fp32-level tie
            assert list(idx[r]) == list(want), (r, idx[r], want)
        assert np.abs(val[r] - p[idx[r]]).max() < 1e-5


def test_sampler_distribution():
    nu, ni, m_neg = 50, 200, 3
    rs = np.random.RandomState(2)
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, 20), replace=False)).astype(np.int32) for _ in range(nu)]
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    u, i, y = ops.neumf_sample(nu, ni, torch.from_numpy(indptr).to(DEV), torch.from_numpy(np.concatenate(rows)).to(DEV), m_neg, 7)
    u, i, y = u.cpu().numpy(), i.cpu().numpy(), y.cpu().numpy()
    nnz = int(indptr[-1])
    assert len(u) == nnz * (1 + m_neg) and y.sum() == nnz
    pos = {(a, b) for a, b, l in zip(u, i, y) if l == 1}
    assert pos == {(uu, int(it)) for uu in range(nu) for it in rows[uu]}
    for a, b, l in zip(u, i, y):
        if l == 0:
            assert b not in set(rows[a].tolist())


def test_neumf_yaml_trains(tmp_path):
    import os, yaml
    from elliot_b200 import run_experiment
    g = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bprmf_small.npz")))
    for name in ("train", "test"):
        with open(tmp_path / f"{name}.tsv", "w") as fh:
            for a, b, r in g[name]:
                fh.write(f"{int(a)}\t{int(b)}\t{r}\n")

    def cfg(epochs, lr):
        c = {"experiment": {"dataset": "golden", "data_config": {"strategy": "fixed", "train_path": "train.tsv", "test_path": "test.tsv"},
                            "top_k": 10, "evaluation": {"simple_metrics": ["nDCG"]},
                            "path_output_rec_result": "o/r", "path_output_rec_weight": "o/w", "path_output_rec_performance": "o/p",
                            "models": {"NeuMF": {"meta": {}, "epochs": epochs, "batch_size": 1024, "mf_factors": 16, "lr": lr, "m": 4}}}}
        p = tmp_path / "c.yml"; p.write_text(yaml.safe_dump(c)); return str(p)
    r0 = run_experiment(cfg(1, 0.0))
    r1 = run_experiment(cfg(30, 0.003))
    assert r1[0]["test_results"][10]["nDCG"] > 1.5 * r0[0]["test_results"][10]["nDCG"] + 0.02


def test_sharded_model_at_world_1_tracks_the_ordinary_model():
    """recommender/neumf_sharded.py (row-sharded item tables, SURVEY.md §8e) with no process group: every all-to-all
    degenerates to a copy, so the step must equal the ordinary model's (same kernels on fetched row copies)."""
    from elliot_b200.recommender.neumf import NeuralMatrixFactorizationModel
    from elliot_b200.recommender.neumf_sharded import ShardedNeuMFModel
    dev = torch.device(DEV)
    NU, NI, F, B = 5000, 3000, 64, 4096                       # the configuration of tools/neumf_sharded_w1.py
    sh = ShardedNeuMFModel(NU, NI, F, 1e-3, 42, dev); ref = NeuralMatrixFactorizationModel(NU, NI, F, 1e-3, 42, dev)
    g = torch.Generator(device=dev); g.manual_seed(1)
    for s in range(3):
        u = torch.randint(0, NU, (B,), device=dev, generator=g, dtype=torch.int32)
        it = torch.randint(0, NI, (B,), device=dev, generator=g, dtype=torch.int32)
        y = (torch.rand(B, device=dev, generator=g) < 0.3).float()
        la, lb = sh.train_step((u, it, y)).item(), ref.train_step((u, it, y)).item()
        assert abs(la - lb) < 1e-6 * abs(lb)
    rel = lambda a, b: float((a - b).norm() / b.norm().clamp_min(1e-12))
    assert rel(sh.P["U_mf"], ref.P["U_mf"]) < 1e-5 and rel(sh.P["U_mlp"], ref.P["U_mlp"]) < 1e-5
    assert rel(sh.P["I"][:, :F], ref.P["I_mf"]) < 1e-5 and rel(sh.P["I"][:, F:], ref.P["I_mlp"]) < 1e-5
    for k in ("W1", "W2", "W3", "wp"):
        assert rel(sh.P[k], ref.P[k]) < 1e-5, k


def test_train_step_wiring_is_exact_with_the_fp32_checking_gemm():
    """Same comparison with the dense layers on the fp32 checking GEMM (ops.exact_gemm): without bf16 rounding every gradient
    of the step agrees with the fp64 restatement to 1e-4 (fp32 accumulation) — the wiring of the 9 GEMMs, the ReLU masks, the
    head and the embedding scatter is what the model code says, not merely "close"."""
    nu, ni, f, B = 120, 90, 16, 700
    with ops.exact_gemm():
        m = NeuralMatrixFactorizationModel(nu, ni, f, 1e-3, 42, DEV)
        for k in ("b1", "b2", "b3", "bp"):
            m.P[k].normal_(0, 0.05)
        for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
            m.P[k].mul_(4.0)
        m._refresh()
        P = _ref_params(m)
        rs = np.random.RandomState(0)
        u = rs.randint(0, nu, B).astype(np.int32); i = rs.randint(0, ni, B).astype(np.int32)
        y = (rs.rand(B) < 0.3).astype(np.float32)
        loss_ref, G, _ = tfm.neumf_forward_backward(P, u, i, y.astype(np.float64))
        loss = m.train_step((torch.from_numpy(u).to(DEV), torch.from_numpy(i).to(DEV), torch.from_numpy(y).to(DEV))).item()
    assert abs(loss - loss_ref) < 1e-5 * abs(loss_ref)
    rel = lambda a, b: np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12)
    M = lambda k: m.M[k].double().cpu().numpy() / 0.1         # first Adam step: m = 0.1 g
    for k in ("W3", "W2", "W1"):
        assert rel(M(k), G[k].T) < 1e-4, (k, rel(M(k), G[k].T))
    for k, n in (("b3", f), ("b2", 2 * f), ("b1", 4 * f)):
        assert rel(M(k)[:n], G[k]) < 1e-4, k
    assert rel(M("wp"), G["wp"]) < 1e-4 and abs(M("bp")[0] - G["bp"]) < 1e-4 * abs(G["bp"]) + 1e-7
    for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
        assert rel(M(k), G[k]) < 1e-4, (k, rel(M(k), G[k]))
