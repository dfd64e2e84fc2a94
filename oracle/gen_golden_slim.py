#!/usr/bin/env python
"""Mint the SLIM goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/slim_cases.npz
      the reference's `SlimModel` (latent_factor_models/Slim/slim_model.py), imported by file path, on synthetic rating
      matrices: ratings 1-5, implicit ones and half stars; (alpha, l1_ratio, neighborhood) in {(0.0788, 1.19e-5, 544)
      (recsys_config.yml's block: the min(nnz - 1, neighborhood) rule drops a coefficient), (0.001, 0.001, 10) (the
      defaults), (0.05, 0.5, 20) (screening excludes features)}; a user without ratings and a duplicated item in every
      case, a cold item in some, and num_items == num_users once.  A pass-through wrapper on ElasticNet.fit records each
      item's coef_, n_iter_ and dual_gap_.  Recorded per case: those, W (the reference's float32 csr_matrix), the
      SHA-256 of its dense float32 preds and the top-k lists of its get_user_recs.  sklearn's version is recorded: the
      solver is sklearn's, not the reference's pinned 0.24.1.
  tests/golden/slim_c1.npz
      elliot.run.run_experiment on config_files/recsys_config.yml's Slim block (l1_ratio 0.0000119, alpha 0.0788,
      neighborhood 544, save_recs) over the C1 synthetic file of elliot_b200/synth_c1.py: test metrics, the stored rec
      file's name and the lists of its first 400 users, the dataset checksum, the wall time.

Every synthetic case is also checked against oracle/slim.py here (the checks tests/test_oracle_slim.py makes).

    python oracle/gen_golden_slim.py [--skip-c1] [--skip-cases]
"""
import argparse
import os
import sys
import warnings

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs  # noqa: E402
from oracle.rp3beta import preds_digest  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 10
SEED = 42
# name: (users, items, rating kind, alpha, l1_ratio, neighborhood, cold item, seed)
CASES = {
    "int_tois": (300, 200, "int", 0.0788, 1.19e-5, 544, True, 1),
    "implicit_default": (250, 150, "implicit", 0.001, 0.001, 10, False, 2),
    "half_screen": (200, 120, "half", 0.05, 0.5, 20, True, 3),
    "int_square_tois": (120, 120, "int", 0.0788, 1.19e-5, 544, False, 4),
    "implicit_screen": (150, 100, "implicit", 0.05, 0.5, 20, False, 5),
    "half_default": (180, 140, "half", 0.001, 0.001, 10, False, 6),
}


class _Data:
    """The DataSet fields SlimModel reads; public ids == private ids."""

    def __init__(self, R):
        U, I = R.shape
        self.sp_i_train_ratings = sp.csr_matrix(R.astype(np.float32))
        self.num_users, self.num_items = U, I
        self.users, self.items = list(range(U)), list(range(I))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}


def matrix(U, I, kind, cold, seed):
    g = np.random.default_rng(seed)
    dens = g.random((U, I)) < 0.05 + 0.3 * g.random(I)[None, :] ** 3      # uneven item popularity
    if kind == "half":
        vals = g.integers(1, 11, (U, I)) / 2.0
    elif kind == "implicit":
        vals = np.ones((U, I))
    else:
        vals = g.integers(1, 6, (U, I)).astype(np.float64)
    R = np.where(dens, vals, 0.0)
    if cold:
        R[:, I - 2] = 0                                   # a cold item: no coefficients, an empty column of W
    R[U - 3, :] = 0                                       # a user without ratings
    R[:, 1] = R[:, 0]                                     # a duplicated item: exact ties
    return R


def reference_case(mod, R, alpha, l1_ratio, nbh):
    data = _Data(R)
    got = {"coef": [], "n_iter": [], "gap": []}
    real_fit = mod.ElasticNet.fit

    def recording_fit(self, X, y, *a, **k):              # pass-through: records what sklearn computed
        out = real_fit(self, X, y, *a, **k)
        got["coef"].append(np.asarray(self.coef_, np.float32).copy())
        got["n_iter"].append(int(self.n_iter_))
        got["gap"].append(float(self.dual_gap_))
        return out
    mod.ElasticNet.fit = recording_fit
    try:
        m = mod.SlimModel(data, data.num_users, data.num_items, l1_ratio, alpha, 1, nbh, SEED)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m.train(False)
    finally:
        mod.ElasticNet.fit = real_fit
    W = m._w_sparse.tocsr()
    W.sort_indices()
    m.prepare_predictions()
    preds = np.asarray(m.pred_mat)
    assert preds.dtype == np.float32
    mask = R == 0
    ti = np.full((R.shape[0], TOPK), -1, np.int64)
    for u in data.users:
        recs = m.get_user_recs(u, mask, TOPK)
        ti[u, :len(recs)] = [int(i) for i, _ in recs]
    return {"coef": np.array(got["coef"], np.float32), "n_iter": np.array(got["n_iter"], np.int32),
            "gap": np.array(got["gap"], np.float64), "w_data": W.data.astype(np.float32),
            "w_indices": W.indices.astype(np.int32), "w_indptr": W.indptr.astype(np.int64),
            "preds_sha256": np.array(preds_digest(preds)), "topk_idx": ti.astype(np.int16)}


def synthetic(ref_root):
    import sklearn
    from oracle.slim import check_case
    ref_stubs.install()
    mod = ref_stubs.load(os.path.join(ref_root, "elliot/recommender/latent_factor_models/Slim/slim_model.py"), "ref_slim_model")
    out = {"cases": np.array(list(CASES)), "topk": TOPK, "seed": SEED, "sklearn_version": np.array(sklearn.__version__)}
    for name, (U, I, kind, alpha, l1_ratio, nbh, cold, seed) in CASES.items():
        R = matrix(U, I, kind, cold, seed)
        got = reference_case(mod, R, alpha, l1_ratio, nbh)
        out.update({f"{name}_R": R.astype(np.float16), f"{name}_alpha": alpha, f"{name}_l1_ratio": l1_ratio,
                    f"{name}_neighborhood": nbh})
        out.update({f"{name}_{k}": v for k, v in got.items()})
        print(name, check_case(out, name), flush=True)
    np.savez_compressed(os.path.join(GOLD, "slim_cases.npz"), **out)


def c1_run():
    import sklearn
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got, recs, checksum, dt = ref_stubs.run_c1(synth_c1.slim_yaml)
    assert len(recs) == 1, list(recs)
    (name, rec), = recs.items()
    np.savez_compressed(os.path.join(GOLD, "slim_c1.npz"), metrics=np.array(ref_stubs.METRICS),
                        test_metrics=np.array(got[-1]), rec_file=name, checksum=np.uint64(checksum), reference_seconds=dt,
                        sklearn_version=np.array(sklearn.__version__), **ref_stubs.first_users(rec))
    print(f"slim_c1: metrics {dict(zip(ref_stubs.METRICS, got[-1]))}, reference run {dt:.0f} s, {name}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    ap.add_argument("--skip-cases", action="store_true")
    args = ap.parse_args()
    if not args.skip_cases:
        synthetic(ref_stubs.REF)
    if not args.skip_c1:
        c1_run()


if __name__ == "__main__":
    main()
