#!/usr/bin/env python
"""Mint golden vectors from the REFERENCE's own code (needs a checkout of the original project).

The reference ships no tests/golden vectors (SURVEY.md §4).  This script imports
  elliot/dataset/samplers/custom_sampler.py            (Sampler)
  elliot/recommender/latent_factor_models/BPRMF/BPRMF_model.py   (MFModel)
  elliot.dataset.dataset.DataSet, elliot.evaluation.evaluator.Evaluator
from the original project (REF below, read-only), runs them unmodified on small seeded synthetic
data and writes tests/golden/bprmf_<case>.npz.  The tests need no copy of the original project:
they only ever read the committed .npz files.

    python oracle/gen_golden.py            # rewrites tests/golden/*.npz
"""
import importlib.util
import logging
import os
import sys
from types import SimpleNamespace

import numpy as np
import pandas as pd

# a checkout of the original Elliot project: $ELLIOT_REFERENCE, or a directory named `reference` beside this repository
REF = os.environ.get("ELLIOT_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def synth(n_users, n_items, mean_pos, seed, id_stride_u=3, id_stride_i=7):
    """Seeded implicit-feedback interactions with non-contiguous public ids, a
    popularity skew, one single-item user (randint(1) draws nothing) and one
    heavy user."""
    g = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.8
    pop /= pop.sum()
    rows = []
    for u in range(n_users):
        if u == 1:
            c = 1
        elif u == 2:
            c = min(n_items - 3, 6 * mean_pos)
        else:
            c = int(np.clip(g.lognormal(np.log(mean_pos), 0.6), 2, n_items // 2))
        its = g.choice(n_items, size=c, replace=False, p=pop)
        for it in its:
            rows.append((10 + id_stride_u * u, 100 + id_stride_i * int(it)))
    rows = np.array(rows, dtype=np.int64)
    g.shuffle(rows)
    # 80/20 hold-out per user (at least one train item)
    train, test = [], []
    byu = {}
    for u, i in rows:
        byu.setdefault(int(u), []).append(int(i))
    for u, its in byu.items():
        n_te = len(its) // 5
        for q, i in enumerate(its):
            (test if q < n_te else train).append((u, i, 1.0))
    return np.array(train), np.array(test)


def make_case(name, n_users, n_items, mean_pos, d, seed_data, model_seed, epochs, k):
    sys.path.insert(0, REF)
    logging.disable(logging.CRITICAL)
    cs = _load("ref_custom_sampler", "elliot/dataset/samplers/custom_sampler.py")
    mf = _load("ref_bprmf_model", "elliot/recommender/latent_factor_models/BPRMF/BPRMF_model.py")
    import elliot.dataset.dataset as ds
    from elliot.evaluation.evaluator import Evaluator

    train, test = synth(n_users, n_items, mean_pos, seed_data)
    cols = ["userId", "itemId", "rating"]
    tr = pd.DataFrame({"userId": train[:, 0].astype(np.int64), "itemId": train[:, 1].astype(np.int64),
                       "rating": train[:, 2]})
    te = pd.DataFrame({"userId": test[:, 0].astype(np.int64), "itemId": test[:, 1].astype(np.int64),
                       "rating": test[:, 2]})
    config = SimpleNamespace(config_test=True, align_side_with_train=False, top_k=k,
                             evaluation=SimpleNamespace(simple_metrics=["nDCG", "HR", "Precision", "Recall"],
                                                        relevance_threshold=0, paired_ttest=False, cutoffs=[k]))
    data = ds.DataSet(config, (tr, te), SimpleNamespace())

    users = np.array(data.users, dtype=np.int64)      # private -> public
    items = np.array(data.items, dtype=np.int64)

    # M0: init (BPRMF_model.py:15-56).  Construction order in BPRMF.__init__ (BPRMF.py:83-91):
    # MFModel first (seeds np.random with the model seed), Sampler second (reseeds 42).
    lr, ru, rb, rp, rn = 0.05, 0.0025, 0.0, 0.0025, 0.00025
    model = mf.MFModel(d, data, lr, ru, rb, rp, rn, model_seed)
    U0 = model._user_factors.copy(); V0 = model._item_factors.copy()
    sampler = cs.Sampler(data.i_train_dict)

    ui_indptr = np.zeros(len(users) + 1, dtype=np.int64)
    ui_list = []
    for u in range(len(users)):
        ui_list.extend(sampler._ui_dict[u])
        ui_indptr[u + 1] = len(ui_list)
    ui_indices = np.array(ui_list, dtype=np.int32)

    tu, ti, tj = [], [], []
    snapshots = {}
    T = data.transactions
    for ep in range(epochs):
        for batch in sampler.step(T, 1):
            tu.append(int(batch[0][0, 0])); ti.append(int(batch[1][0, 0])); tj.append(int(batch[2][0, 0]))
            model.train_step(batch)
        if ep == 0:
            snapshots["U_ep1"] = model._user_factors.copy()
            snapshots["V_ep1"] = model._item_factors.copy()
            snapshots["b_ep1"] = model._item_bias.copy()
    # draws that follow the last triple: pins the stream position after `epochs` epochs
    tail = np.array([np.random.randint(1 << 20) for _ in range(4)], dtype=np.int64)

    mask = data.allunrated_mask
    rec_idx = np.full((len(users), k), -1, dtype=np.int32)
    rec_val = np.full((len(users), k), -np.inf)
    recs = {}
    for pu, u_pub in enumerate(data.users):
        r = model.get_user_predictions(u_pub, mask, k)
        recs[u_pub] = r
        for q, (it, sc) in enumerate(r):
            rec_idx[pu, q] = data.public_items[it]
            rec_val[pu, q] = sc
    params = SimpleNamespace(meta=SimpleNamespace())
    ev = Evaluator(data, params)
    res = ev.eval((recs, recs))
    metrics = res[k]["test_results"]

    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(
        os.path.join(OUT, f"bprmf_{name}.npz"),
        train=train, test=test, users=users, items=items, d=d, model_seed=model_seed, k=k, epochs=epochs,
        hp=np.array([lr, ru, rb, rp, rn]), transactions=T,
        ui_indptr=ui_indptr, ui_indices=ui_indices,
        tu=np.array(tu, np.int32), ti=np.array(ti, np.int32), tj=np.array(tj, np.int32), tail=tail,
        U0=U0, V0=V0, U=model._user_factors, V=model._item_factors, b=model._item_bias,
        rec_idx=rec_idx, rec_val=rec_val,
        metric_names=np.array(sorted(metrics.keys())), metric_vals=np.array([metrics[m] for m in sorted(metrics.keys())]),
        **snapshots)
    print(name, "users", len(users), "items", len(items), "T", T, "triples", len(tu), {m: round(v, 6) for m, v in metrics.items()})


def make_split_case():
    """Reference Splitter (base_splitter.py:62-111,256-274) on a small frame: pins the split stream."""
    sys.path.insert(0, REF)
    from elliot.splitter.base_splitter import Splitter
    g = np.random.default_rng(5)
    rows = []
    for u in g.permutation(40):
        for it in g.choice(60, size=int(g.integers(3, 15)), replace=False):
            rows.append((int(u) * 2 + 1, int(it) + 500, 1.0))
    rows = np.array(rows)
    g.shuffle(rows)
    df = pd.DataFrame({"userId": rows[:, 0].astype(np.int64), "itemId": rows[:, 1].astype(np.int64), "rating": rows[:, 2]})
    ns = SimpleNamespace(test_splitting=SimpleNamespace(strategy="random_subsampling", test_ratio=0.2))
    (train, test), = Splitter(df.copy(), ns, 42).process_splitting()
    np.savez_compressed(os.path.join(OUT, "split_random_subsampling.npz"), data=rows,
                        train=train[["userId", "itemId", "rating"]].to_numpy(),
                        test=test[["userId", "itemId", "rating"]].to_numpy())
    print("split", len(df), len(train), len(test))


def make_sampler_cases():
    """Reference NeuMF pointwise sampler (neural/NeuMF/custom_sampler.py:14-48) and the autoencoder row sampler
    (dataset/samplers/sparse_sampler.py:9-25) on the tiny case: pins epoch sample order / user-batch order."""
    import scipy.sparse as sp
    ns = _load("ref_neumf_sampler", "elliot/recommender/neural/NeuMF/custom_sampler.py")
    ss = _load("ref_sparse_sampler", "elliot/dataset/samplers/sparse_sampler.py")
    g = np.load(os.path.join(OUT, "bprmf_tiny.npz"))
    nu = len(g["users"])
    i_train = {u: {int(i): 1.0 for i in g["ui_indices"][g["ui_indptr"][u]:g["ui_indptr"][u + 1]]} for u in range(nu)}
    out = {}
    for m in (0, 3):
        smp = ns.Sampler(i_train, m)
        eps = []
        for ep in range(2):
            u, i, b = [], [], []
            for bu, bi, bb in smp.step(64):
                u.extend(bu.tolist()); i.extend(bi.tolist()); b.extend(bb.tolist())
            eps.append(np.array([u, i, b], dtype=np.int64))
        out[f"neumf_m{m}_ep0"], out[f"neumf_m{m}_ep1"] = eps
    rows = [u for u in range(nu) for _ in i_train[u]]; cols = [i for u in range(nu) for i in i_train[u]]
    mat = sp.csr_matrix((np.ones(len(rows), dtype=np.float32), (rows, cols)), shape=(nu, len(g["items"])))
    vs = ss.Sampler(mat)
    order = []
    for ep in range(2):
        ep_rows = []
        for batch in vs.step(nu, 16):
            # recover the user of each dense row from its item pattern (rows are unique in this case)
            ep_rows.append(batch.shape[0])
        order.append(ep_rows)
    import random
    random.seed(42)
    perm = [random.sample(range(nu), nu) for _ in range(2)]            # what sparse_sampler.py:18 draws, epoch by epoch
    # cross-check against the reference's dense batches
    vs2 = ss.Sampler(mat)
    for ep in range(2):
        got = np.concatenate([b for b in vs2.step(nu, 16)])
        assert np.array_equal(got, mat[perm[ep]].toarray())
    out["vae_perm"] = np.array(perm, dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "samplers_tiny.npz"), **out)
    print("samplers", {k: v.shape for k, v in out.items()})


def make_mf2020_case(name, d, seed, m, epochs, lr, reg, k):
    """Reference MF2020 (latent_factor_models/MF2020/MF_model.py + custom_sampler_rendle.py) on the train/test split
    of bprmf_<name>.npz, with the construction order of MF.py:58-80 under @init_charger
    (base_recommender_model.py:149-150): seed np/random -> Sampler (seeds again) -> MFModel (seeds np, draws the
    tables) -> epochs of sampler.step(100000) / train_step."""
    import random
    sys.path.insert(0, REF)
    logging.disable(logging.CRITICAL)
    ps = _load("ref_mf2020_sampler", "elliot/recommender/latent_factor_models/MF2020/custom_sampler_rendle.py")
    mm = _load("ref_mf2020_model", "elliot/recommender/latent_factor_models/MF2020/MF_model.py")
    import elliot.dataset.dataset as ds
    from elliot.evaluation.evaluator import Evaluator
    g = np.load(os.path.join(OUT, f"bprmf_{name}.npz"))
    f = lambda a: pd.DataFrame({"userId": a[:, 0].astype(np.int64), "itemId": a[:, 1].astype(np.int64), "rating": a[:, 2]})
    config = SimpleNamespace(config_test=True, align_side_with_train=False, top_k=k,
                             evaluation=SimpleNamespace(simple_metrics=["nDCG", "HR", "Precision", "Recall"],
                                                        relevance_threshold=0, paired_ttest=False, cutoffs=[k]))
    data = ds.DataSet(config, (f(g["train"]), f(g["test"])), SimpleNamespace())
    np.random.seed(seed); random.seed(seed)                                   # init_charger
    sampler = ps.Sampler(data.i_train_dict, m, data.sp_i_train, seed)
    model = mm.MFModel(d, data, lr, reg, seed)
    U0, V0 = model._user_factors.copy(), model._item_factors.copy()
    pos = np.array([(int(a), int(b)) for a, b, _ in sampler._positive_pairs], dtype=np.int32)
    samples, batch_losses, epoch_loss = [], [], []
    for ep in range(epochs):
        loss, ep_rows, bl = 0.0, [], []
        for batch in sampler.step(100000):
            ep_rows.append(batch.copy())
            s = model.train_step(batch)
            bl.append(float(s)); loss += s / len(batch)
        samples.append(np.concatenate(ep_rows)); batch_losses.append(np.array(bl)); epoch_loss.append(loss)
    model.prepare_predictions()
    mask = data.allunrated_mask
    rec_idx = np.full((len(data.users), k), -1, dtype=np.int32); rec_val = np.full((len(data.users), k), -np.inf)
    recs = {}
    for pu, u_pub in enumerate(data.users):
        r = model.get_user_predictions(u_pub, mask, k)
        recs[u_pub] = r
        for q, (it, sc) in enumerate(r):
            rec_idx[pu, q] = data.public_items[it]; rec_val[pu, q] = sc
    metrics = Evaluator(data, SimpleNamespace(meta=SimpleNamespace())).eval((recs, recs))[k]["test_results"]
    out = {f"samples_ep{e}": samples[e] for e in range(epochs)}
    out.update({f"batch_loss_ep{e}": batch_losses[e] for e in range(epochs)})
    np.savez_compressed(os.path.join(OUT, f"mf2020_{name}.npz"), d=d, seed=seed, m=m, epochs=epochs, lr=lr, reg=reg, k=k,
                        positives=pos, U0=U0, V0=V0, U=model._user_factors, V=model._item_factors,
                        ub=model._user_bias, ib=model._item_bias, gb=model._global_bias, epoch_loss=np.array(epoch_loss),
                        rec_idx=rec_idx, rec_val=rec_val, metric_names=np.array(sorted(metrics)),
                        metric_vals=np.array([metrics[x] for x in sorted(metrics)]), **out)
    print("mf2020", name, "samples/epoch", len(samples[0]), "gb", model._global_bias, {x: round(v, 6) for x, v in metrics.items()})


if __name__ == "__main__":
    make_split_case()
    make_case("tiny", n_users=60, n_items=48, mean_pos=8, d=10, seed_data=1, model_seed=42, epochs=2, k=10)
    make_sampler_cases()
    make_case("small", n_users=400, n_items=300, mean_pos=20, d=64, seed_data=2, model_seed=7, epochs=2, k=10)
    make_mf2020_case("tiny", d=10, seed=42, m=2, epochs=2, lr=0.05, reg=0.01, k=10)
    make_mf2020_case("small", d=64, seed=7, m=3, epochs=2, lr=0.05, reg=0.005, k=10)
