#!/usr/bin/env python
"""Mint the EASE^R goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/ease_cases.npz
      the reference's `EASER` class (autoencoders/EASE_R/ease_r.py), imported by file path, on synthetic rating matrices:
      ratings 1-5 (an indefinite normal matrix), implicit ones (positive definite) and half stars; l2_norm in
      {1e3, 10, 0.3}; a cold item, a user without ratings and a duplicated item (near-ties) in every case; up to 300
      items, so the blocked inverse spans several panels.  The instance is made without `init_charger` (it needs a whole
      experiment configuration) and given only the fields `train()` and `get_user_predictions()` read; its `evaluate`
      is a no-op, because these cases record the model, not metrics.  Recorded per case: the reference's float32
      preds and its top-k lists from `get_user_predictions`.
  tests/golden/ease_c1.npz
      elliot.run.run_experiment on an EASER block (defaults, save_recs) over the C1 synthetic file of
      elliot_b200/synth_c1.py (oracle/ref_stubs.py harness, as gen_golden_knn.py): test metrics, the stored rec file's
      name and the lists of its first 400 users, the dataset checksum, the wall time.

Every synthetic case is also checked against the fp64 restatement oracle/ease.py: preds within 1e-5 of max |preds|
and the top-k lists equal at every isolated rank.

    python oracle/gen_golden_ease.py [--skip-c1]
"""
import argparse
import logging
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ease as oease, ref_stubs  # noqa: E402
from oracle.knn import isolated  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 10
# name: (users, items, rating kind, l2_norm, seed)
CASES = {
    "int_l1000": (200, 300, "int", 1e3, 1),
    "int_l10": (150, 130, "int", 10.0, 2),
    "implicit_l1000": (200, 300, "implicit", 1e3, 3),
    "implicit_l0.3": (150, 200, "implicit", 0.3, 4),
    "half_l10": (160, 257, "half", 10.0, 5),
    "half_l0.3": (60, 40, "half", 0.3, 6),
    "int_l0.3_tiny": (40, 25, "int", 0.3, 7),
}


class _Data:
    """The DataSet fields the reference's EASER reads; public ids == private ids."""

    def __init__(self, R):
        U, I = R.shape
        self.sp_i_train_ratings = sp.csr_matrix(R.astype(np.float32))
        self.num_users, self.num_items = U, I
        self.users, self.items = list(range(U)), list(range(I))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}
        self.train_dict = {u: {int(i): float(R[u, i]) for i in np.flatnonzero(R[u])} for u in self.users}


def _matrix(U, I, kind, seed):
    g = np.random.default_rng(seed)
    dens = g.random((U, I)) < 0.12 + 0.3 * g.random(I)[None, :] ** 3      # uneven item popularity
    if kind == "half":
        vals = g.integers(1, 11, (U, I)) / 2.0
    elif kind == "implicit":
        vals = np.ones((U, I))
    else:
        vals = g.integers(1, 6, (U, I)).astype(np.float64)
    R = np.where(dens, vals, 0.0)
    R[:, I - 2] = 0                                       # a cold item
    R[U - 3, :] = 0                                       # a user without ratings
    R[:, 1] = R[:, 0]                                     # a duplicated item: near-ties in every user's scores
    return R


def _reference_case(mod, R, l2_norm):
    data = _Data(R)
    m = mod.EASER.__new__(mod.EASER)
    m._data, m._l2_norm, m._neighborhood, m._restore = data, float(l2_norm), data.num_items, False
    m.logger = logging.getLogger("ease_golden")
    m.evaluate = lambda *a, **k: None
    m.train()
    preds = np.array(m._preds, dtype=np.float32)          # before get_user_predictions writes -inf into it
    mask = R == 0
    ti = np.full((R.shape[0], TOPK), -1, np.int64)
    tv = np.full((R.shape[0], TOPK), -np.inf)
    for u in data.users:
        recs = m.get_user_predictions(u, mask, TOPK)
        recs = [(i, v) for i, v in recs if np.isfinite(v)]  # the reference pads with masked (-inf) items
        ti[u, :len(recs)] = [int(i) for i, _ in recs]
        tv[u, :len(recs)] = [float(v) for _, v in recs]
    return preds, ti, tv


def synthetic(ref_root):
    ref_stubs.install()
    mod = ref_stubs.load(os.path.join(ref_root, "elliot/recommender/autoencoders/EASE_R/ease_r.py"), "ref_ease_r")
    out = {"cases": np.array(list(CASES)), "topk": TOPK}
    for name, (U, I, kind, lam, seed) in CASES.items():
        R = _matrix(U, I, kind, seed)
        P, ti, tv = _reference_case(mod, R, lam)
        _, Po, oi, ov = oease.run(R, lam, TOPK + 1)
        scale = np.abs(P).max()
        err = np.abs(Po - P).max() / scale
        assert err < 1e-5, (name, err)
        iso = isolated(ov[:, :TOPK], ov[:, TOPK]) & np.isfinite(tv)
        assert np.array_equal(oi[:, :TOPK][iso], ti[iso]), name
        assert np.array_equal(np.isfinite(tv), oi[:, :TOPK] >= 0), name
        out.update({f"{name}_R": R.astype(np.float16), f"{name}_l2_norm": lam, f"{name}_preds": P, f"{name}_topk_idx": ti,
                    f"{name}_topk_val": tv})
        print(f"{name}: oracle preds within {err:.1e} of max |preds|, {iso.mean():.3f} of ranks isolated", flush=True)
    np.savez_compressed(os.path.join(GOLD, "ease_cases.npz"), **out)


def c1_run():
    got, recs, checksum, dt = ref_stubs.run_c1(synth_c1.ease_yaml)
    assert len(recs) == 1, list(recs)
    (name, rec), = recs.items()
    np.savez_compressed(os.path.join(GOLD, "ease_c1.npz"), metrics=np.array(ref_stubs.METRICS),
                        test_metrics=np.array(got[-1]), rec_file=name, checksum=np.uint64(checksum), reference_seconds=dt,
                        **ref_stubs.first_users(rec))
    print(f"ease_c1: metrics {dict(zip(ref_stubs.METRICS, got[-1]))}, reference run {dt:.0f} s, {name}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    args = ap.parse_args()
    synthetic(ref_stubs.REF)
    if not args.skip_c1:
        c1_run()


if __name__ == "__main__":
    main()
