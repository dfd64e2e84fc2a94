#!/usr/bin/env python
"""Mint the PureSVD goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/pure_svd_cases.npz
      the reference's own `PureSVDModel` (latent_factor_models/PureSVD/pure_svd_model.py), imported by file path, on
      small synthetic binary matrices, each with an item without entries, a user without entries and a duplicated item.
      The cases cover both orientations (more users than items and the reverse), 7 and 4 power iterations, factors 10 and
      190 (the largest this build takes), factors + 10 > min(U, I), and factors > min(U, I).  Recorded per case: R, the
      factors, user_vec, item_vec, the singular values of the same randomized_svd call, and the top-k lists of
      `get_user_recs`.  Before saving, every case is checked against the fp64 restatement oracle/pure_svd.py
      (oracle.pure_svd.check_against).
  tests/golden/pure_svd_c1.npz
      elliot.run.run_experiment on synth_c1.pure_svd_yaml over the C1 synthetic file (oracle/ref_stubs.py harness): the
      test metrics, the rec file's name and its first 400 users' lists, the dataset checksum and the wall time.

The sklearn version is recorded in both files.

    python oracle/gen_golden_pure_svd.py [--skip-c1]
"""
import argparse
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import pure_svd as opsvd, ref_stubs  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 10
SEED = 42
# name: (users, items, factors, density)
CASES = {
    "tall_f10_it7": (300, 150, 10, 0.08),
    "wide_f10_it7": (150, 300, 10, 0.08),
    "tall_f10_it4": (120, 60, 10, 0.2),
    "tall_f190": (420, 260, 190, 0.1),
    "wide_w_over_min": (40, 70, 35, 0.25),
    "tall_f_over_min": (60, 30, 40, 0.3),
}


class _Data:
    """The DataSet fields the reference's PureSVDModel reads; public ids == private ids."""

    def __init__(self, R):
        U, I = R.shape
        rows, cols = np.nonzero(R)
        self.sp_i_train = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), dtype=np.float32, shape=(U, I))
        self.num_users, self.num_items = U, I
        self.users, self.items = list(range(U)), list(range(I))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}
        self.train_dict = {u: {int(i): 1.0 for i in np.flatnonzero(R[u])} for u in self.users}


def matrix(seed, U, I, density):
    """Random binary R of about the given density, with skewed item popularity and user activity and a rank-4 taste
    pattern (so that its spectrum decays as real interaction data's does); item I - 1 is cold, user U - 1 has no
    entries and item 1 is a copy of item 0."""
    g = np.random.default_rng(seed)
    pop = (1.0 / np.arange(1, I + 1) ** 0.8)[g.permutation(I)]
    act = g.lognormal(0.0, 0.7, U)
    taste = g.standard_normal((U, 4)) @ g.standard_normal((4, I))
    p = act[:, None] * pop[None, :] * np.exp(0.6 * taste)
    p *= density * U * I / p.sum()
    R = (g.random((U, I)) < p).astype(np.float64)
    R[:, I - 1] = 0
    R[U - 1] = 0
    R[:, 1] = R[:, 0]
    return R


def synthetic(ref_root, sk_version):
    mod = ref_stubs.load(os.path.join(ref_root, "elliot/recommender/latent_factor_models/PureSVD/pure_svd_model.py"),
                         "ref_pure_svd_model")
    from sklearn.utils.extmath import randomized_svd
    out = {"cases": np.array(list(CASES)), "topk": TOPK, "seed": SEED, "sklearn_version": sk_version}
    for name, (U, I, f, dens) in CASES.items():
        R = matrix(1, U, I, dens)
        data = _Data(R)
        m = mod.PureSVDModel(f, data, SEED)
        m.train_step()
        _, s, _ = randomized_svd(data.sp_i_train, n_components=f, random_state=SEED)
        user_vec, item_vec = np.asarray(m.user_vec), np.asarray(m.item_vec)
        assert np.allclose(np.sqrt((item_vec.astype(np.float64) ** 2).sum(0)), s, rtol=1e-4, atol=1e-5 * s[0]), name
        mask = R == 0
        ti = np.full((U, TOPK), -1, np.int64)
        tv = np.full((U, TOPK), -np.inf)
        for u in range(U):
            recs = m.get_user_recs(u, mask, TOPK)
            ti[u, :len(recs)] = [int(i) for i, _ in recs]
            tv[u, :len(recs)] = [float(v) for _, v in recs]
        case = {"R": R, "s": s, "user_vec": user_vec, "item_vec": item_vec, "topk_idx": ti}
        ou, oi, os_ = opsvd.fit(R, f, SEED)
        err, n_iso = opsvd.check_against(case, ou, oi, os_)
        out.update({f"{name}_R": R.astype(np.int8), f"{name}_factors": f, f"{name}_user_vec": user_vec,
                    f"{name}_item_vec": item_vec, f"{name}_s": s, f"{name}_topk_idx": ti, f"{name}_topk_val": tv})
        print(f"{name}: {U} x {I}, factors {f}, {len(s)} components; oracle scores within {err:.1e} max|P|, "
              f"{n_iso} isolated ranks equal", flush=True)
    np.savez_compressed(os.path.join(GOLD, "pure_svd_cases.npz"), **out)


def c1_run(sk_version):
    got, recs, checksum, dt = ref_stubs.run_c1(lambda tsv, d, extra: synth_c1.pure_svd_yaml(tsv, d, extra=extra))
    assert len(got) == 1 and len(recs) == 1, (got, list(recs))
    name, rec = list(recs.items())[0]
    out = {"metrics": np.array(ref_stubs.METRICS), "test_metrics": np.array(got[0]), "rec_file": name,
           "checksum": np.uint64(checksum), "reference_seconds": dt, "sklearn_version": sk_version}
    out.update(ref_stubs.first_users(rec))
    np.savez_compressed(os.path.join(GOLD, "pure_svd_c1.npz"), **out)
    print(f"c1: metrics {got[0]}, run {dt:.1f} s, {name}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    args = ap.parse_args()
    import sklearn
    synthetic(ref_stubs.REF, sklearn.__version__)
    if not args.skip_c1:
        c1_run(sklearn.__version__)


if __name__ == "__main__":
    main()
