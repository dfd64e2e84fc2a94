#!/usr/bin/env python
"""Mint the RP3beta goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/rp3beta_cases.npz
      the reference's `RP3beta` class (graph_based/RP3beta/rp3beta.py), imported by file path, on synthetic rating
      matrices: ratings 1-5, implicit ones and half stars; alpha in {1, 1.0807, 0.5}; beta in {0.6, 0.7029, 0};
      normalize_similarity on and off; neighborhood in {10, more than the item count, -1}; a cold item, a user without
      ratings and a duplicated item (exact ties) in every case; at most 300 items.  The instance is made without
      `init_charger` (it needs a whole experiment configuration) and given only the fields `train()` and
      `get_user_predictions()` read; its `evaluate` is a no-op.  Pass-through `csr_matrix` / `csc_matrix` wrappers record
      the similarity lists (rp3beta.py:143) and W (rp3beta.py:173) as the reference builds them.  Recorded per case: those,
      the SHA-256 of the float32 preds (dense, row-major; the
      preds themselves follow bit for bit from R and the recorded W, which the tests check against this digest) and the
      top-k lists of `get_user_predictions`.
  tests/golden/rp3beta_c1.npz
      elliot.run.run_experiment on config_files/recsys_config.yml's RP3beta block (neighborhood 546, alpha 1.0807,
      beta 0.7029, normalize_similarity True, save_recs) over the C1 synthetic file of elliot_b200/synth_c1.py: test
      metrics, the stored rec file's name and the lists of its first 400 users, the dataset checksum, the wall time.

Every synthetic case is also checked against oracle/rp3beta.py here (the same checks tests/test_oracle_rp3beta.py makes).

    python oracle/gen_golden_rp3beta.py [--skip-c1]
"""
import argparse
import logging
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs  # noqa: E402
from oracle.rp3beta import preds_digest  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 10
# name: (users, items, rating kind, alpha, beta, normalize_similarity, neighborhood, seed)
CASES = {
    "int_a1_b0.6_nb10": (150, 300, "int", 1.0, 0.6, False, 10, 1),
    "int_a1.0807_b0.7029_norm_nb546": (90, 100, "int", 1.0807, 0.7029, True, 546, 2),
    "implicit_a0.5_b0_nbm1": (90, 110, "implicit", 0.5, 0.0, False, -1, 3),
    "implicit_a1_b0.6_norm_nb10": (150, 250, "implicit", 1.0, 0.6, True, 10, 4),
    "half_a1.0807_b0.6_norm_nbm1": (80, 129, "half", 1.0807, 0.6, True, -1, 5),
    "half_a0.5_b0.7029_nb10": (120, 180, "half", 0.5, 0.7029, False, 10, 6),
    "int_a0.5_b0_norm_nb400": (60, 40, "int", 0.5, 0.0, True, 400, 7),
    "implicit_a1_b0_nb10": (80, 60, "implicit", 1.0, 0.0, False, 10, 8),
}


class _Data:
    """The DataSet fields the reference's RP3beta reads; public ids == private ids."""

    def __init__(self, R):
        U, I = R.shape
        self.sp_i_train_ratings = sp.csr_matrix(R.astype(np.float32))
        self.num_users, self.num_items = U, I
        self.users, self.items = list(range(U)), list(range(I))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}


def matrix(U, I, kind, seed):
    g = np.random.default_rng(seed)
    dens = g.random((U, I)) < 0.05 + 0.3 * g.random(I)[None, :] ** 3      # uneven item popularity
    if kind == "half":
        vals = g.integers(1, 11, (U, I)) / 2.0
    elif kind == "implicit":
        vals = np.ones((U, I))
    else:
        vals = g.integers(1, 6, (U, I)).astype(np.float64)
    R = np.where(dens, vals, 0.0)
    R[:, I - 2] = 0                                       # a cold item
    R[U - 3, :] = 0                                       # a user without ratings
    R[:, 1] = R[:, 0]                                     # a duplicated item: exact ties
    return R


def reference_case(mod, R, alpha, beta, normalize, nbh):
    data = _Data(R)
    made = {}
    real_csr, real_csc = mod.sparse.csr_matrix, mod.sparse.csc_matrix

    class _Sparse:                                       # pass-through: records the arguments, builds unchanged
        def __getattr__(self, a):
            return getattr(sp, a)

        @staticmethod
        def csr_matrix(arg, **kw):
            made["s"] = arg
            return real_csr(arg, **kw)

        @staticmethod
        def csc_matrix(arg, **kw):
            made["w"] = arg
            return real_csc(arg, **kw)
    m = mod.RP3beta.__new__(mod.RP3beta)
    m._data, m._restore = data, False
    m._neighborhood = data.num_items if nbh == -1 else nbh
    m._alpha, m._beta, m._normalize_similarity = float(alpha), float(beta), bool(normalize)
    m.logger = logging.getLogger("rp3beta_golden")
    m.evaluate = lambda *a, **k: None
    mod.sparse = _Sparse()
    try:
        m.train()
    finally:
        mod.sparse = sp
    s_val, (s_row, s_col) = made["s"]
    w_data, w_rows, w_ptr = (np.asarray(a) for a in made["w"])
    preds = m._preds.toarray()
    assert preds.dtype == np.float32
    mask = R == 0
    ti = np.full((R.shape[0], TOPK), -1, np.int64)
    for u in data.users:
        recs = m.get_user_predictions(u, mask, TOPK)
        recs = [(i, v) for i, v in recs if np.isfinite(v)]  # the reference pads with masked (-inf) items
        ti[u, :len(recs)] = [int(i) for i, _ in recs]
    return {"s_row": np.asarray(s_row, np.int32), "s_col": np.asarray(s_col, np.int32), "s_val": np.asarray(s_val, np.float32),
            "w_data": w_data.astype(np.float32), "w_rows": w_rows.astype(np.int32), "w_ptr": w_ptr.astype(np.int64),
            "preds_sha256": np.array(preds_digest(preds)), "topk_idx": ti.astype(np.int16)}


def synthetic(ref_root):
    from oracle.rp3beta import check_case
    ref_stubs.install()
    mod = ref_stubs.load(os.path.join(ref_root, "elliot/recommender/graph_based/RP3beta/rp3beta.py"), "ref_rp3beta")
    out = {"cases": np.array(list(CASES)), "topk": TOPK}
    for name, (U, I, kind, alpha, beta, norm, nbh, seed) in CASES.items():
        R = matrix(U, I, kind, seed)
        got = reference_case(mod, R, alpha, beta, norm, nbh)
        out.update({f"{name}_R": R.astype(np.float16), f"{name}_alpha": alpha, f"{name}_beta": beta,
                    f"{name}_normalize": norm, f"{name}_neighborhood": nbh})
        out.update({f"{name}_{k}": v for k, v in got.items()})
        print(name, check_case(out, name), flush=True)
    np.savez_compressed(os.path.join(GOLD, "rp3beta_cases.npz"), **out)


def c1_run():
    got, recs, checksum, dt = ref_stubs.run_c1(synth_c1.rp3beta_yaml)
    assert len(recs) == 1, list(recs)
    (name, rec), = recs.items()
    np.savez_compressed(os.path.join(GOLD, "rp3beta_c1.npz"), metrics=np.array(ref_stubs.METRICS),
                        test_metrics=np.array(got[-1]), rec_file=name, checksum=np.uint64(checksum), reference_seconds=dt,
                        **ref_stubs.first_users(rec))
    print(f"rp3beta_c1: metrics {dict(zip(ref_stubs.METRICS, got[-1]))}, reference run {dt:.0f} s, {name}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    args = ap.parse_args()
    synthetic(ref_stubs.REF)
    if not args.skip_c1:
        c1_run()


if __name__ == "__main__":
    main()
