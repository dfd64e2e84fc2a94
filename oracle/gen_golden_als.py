#!/usr/bin/env python
"""Mint the iALS / WRMF goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/als_cases.npz
      the reference's own `iALSModel` and `WRMFModel` (latent_factor_models/iALS/iALS_model.py,
      latent_factor_models/WRMF/wrmf_model.py), imported by file path, each given a FRESH data object (the reference's
      iALS rewrites `sp_i_train` in place), on small synthetic binary matrices with an item without entries.  Cases:
      scaling linear and log (epsilon != 1), non-integer alpha (so the float32 confidences differ from fp64 ones),
      d in {1, 10, 33}, 3 epochs.  Recorded per case: the initial X and Y, X and Y after every epoch, the reference's
      float32 confidence arrays, its top-k lists from `get_user_recs`.
  tests/golden/als_c1.npz
      elliot.run.run_experiment on an iALS block and on a WRMF block (two separate runs) over the C1 synthetic file of
      elliot_b200/synth_c1.py (oracle/ref_stubs.py harness): per-epoch test metrics, the stored rec files' names and the
      lists of the last epoch's first 400 users, the dataset checksum, the wall time and the host time of each `train_step`.

Every synthetic case is also checked against the fp64 restatement oracle/als.py (tables within 1e-12).

    python oracle/gen_golden_als.py [--skip-c1]
"""
import argparse
import importlib
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import als as oals, ref_stubs  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 5
EPOCHS = 3
SEED = 42
# name: (model, d, alpha, epsilon, reg, scaling)
CASES = {
    "ials_lin_d10": ("iALS", 10, 0.37, 1.0, 0.1, "linear"),
    "ials_log_d33": ("iALS", 33, 2.5, 0.3, 0.5, "log"),
    "ials_lin_d1": ("iALS", 1, 1.0, 1.0, 0.1, "linear"),
    "wrmf_d10": ("WRMF", 10, 0.37, None, 0.1, None),
    "wrmf_d33": ("WRMF", 33, 3.0, None, 0.5, None),
    "wrmf_d1": ("WRMF", 1, 1, None, 0.1, None),
}
C1_BLOCKS = {
    "iALS": (3, "      factors: 10\n      alpha: 1\n      epsilon: 1\n      reg: 0.1\n      scaling: linear\n"),
    "WRMF": (2, "      factors: 10\n      alpha: 1\n      reg: 0.1\n"),
}


def _scipy_dense_alias():
    """wrmf_model.py:60 reads `csr_matrix.A`, the dense-array alias that SciPy 1.14 removed; put it back (as
    `toarray()`, what it always was) so the unmodified reference runs on a current SciPy."""
    if not hasattr(sp.spmatrix, "A"):
        sp.spmatrix.A = property(lambda self: self.toarray())


class _Data:
    """The DataSet fields the reference's iALS / WRMF models read; public ids == private ids."""

    def __init__(self, R):
        U, I = R.shape
        rows, cols = np.nonzero(R)
        self.sp_i_train = sp.csr_matrix((np.ones_like(rows), (rows, cols)), dtype="float32", shape=(U, I))
        self.num_users, self.num_items = U, I
        self.users, self.items = list(range(U)), list(range(I))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}
        self.train_dict = {u: {int(i): 1.0 for i in np.flatnonzero(R[u])} for u in self.users}


def _matrix(seed, U=70, I=50):
    g = np.random.default_rng(seed)
    R = (g.random((U, I)) < 0.25).astype(np.float64)
    R[:, I - 3] = 0                                       # an item without train entries
    for u in range(U):                                    # every user has at least one entry
        if not R[u].any():
            R[u, g.integers(0, I - 3)] = 1
    return R


def synthetic(ref_root):
    base = os.path.join(ref_root, "elliot/recommender/latent_factor_models")
    mods = {"iALS": ref_stubs.load(os.path.join(base, "iALS/iALS_model.py"), "ref_ials_model"),
            "WRMF": ref_stubs.load(os.path.join(base, "WRMF/wrmf_model.py"), "ref_wrmf_model")}
    out = {"cases": np.array(list(CASES)), "topk": TOPK, "epochs": EPOCHS}
    for n, (name, (model, d, alpha, eps, reg, scaling)) in enumerate(CASES.items()):
        R = _matrix(100 + n)
        data = _Data(R)                                   # fresh per model: iALS mutates sp_i_train
        mask = data.sp_i_train.toarray() == 0
        np.random.seed(SEED)                              # init_charger (base_recommender_model.py:149)
        if model == "iALS":
            m = mods[model].iALSModel(d, data, np.random, alpha, eps, reg, scaling)
            X0, Y0 = m.X.copy(), m.Y.copy()
            conf = np.array(m.C.data, dtype=np.float32)
        else:
            m = mods[model].WRMFModel(d, data, np.random, alpha, reg)
            X0, Y0 = m.X.toarray(), m.Y.toarray()
            conf = np.array(m.C.data, dtype=np.float32)
        Xs, Ys = [], []
        for _ in range(EPOCHS):
            m.train_step()
            if model == "iALS":
                Xs.append(m.X.copy()); Ys.append(m.Y.copy())
            else:
                Xs.append(m.X.toarray()); Ys.append(m.Y.toarray())
        if model == "iALS":
            m.prepare_predictions()
        U = R.shape[0]
        ti = np.full((U, TOPK), -1, np.int64)
        tv = np.full((U, TOPK), -np.inf)
        for u in range(U):
            recs = m.get_user_recs(u, mask, TOPK)
            ti[u, :len(recs)] = [int(i) for i, _ in recs]
            tv[u, :len(recs)] = [float(v) for _, v in recs]
        mine, (w, c) = oals.train(model, R, X0, Y0, EPOCHS, alpha, reg, eps or 1.0, scaling or "linear")
        err = max(max(np.abs(a - b).max() for a, b in zip(mx, (x, y))) for mx, x, y in zip(mine, Xs, Ys))
        assert err < 1e-12, (name, err)
        oi, _ = oals.topk(mine[-1][0], mine[-1][1], ~mask, TOPK)
        assert np.array_equal(oi, ti), name
        out.update({f"{name}_R": R.astype(np.int8), f"{name}_X0": X0, f"{name}_Y0": Y0, f"{name}_X": np.stack(Xs),
                    f"{name}_Y": np.stack(Ys), f"{name}_conf": conf, f"{name}_topk_idx": ti, f"{name}_topk_val": tv,
                    f"{name}_hp": np.array([d, alpha, eps if eps is not None else np.nan, reg]),
                    f"{name}_scaling": str(scaling)})
        print(f"{name}: oracle tables within {err:.1e} of the reference, top-{TOPK} lists identical", flush=True)
    np.savez_compressed(os.path.join(GOLD, "als_cases.npz"), **out)


def c1_runs():
    ref_stubs.install()
    out = {"metrics": np.array(ref_stubs.METRICS)}
    for model, (epochs, block) in C1_BLOCKS.items():
        mod = importlib.import_module("elliot.recommender.latent_factor_models.iALS.iALS_model" if model == "iALS" else
                                      "elliot.recommender.latent_factor_models.WRMF.wrmf_model")
        cls = mod.iALSModel if model == "iALS" else mod.WRMFModel
        orig_step, steps = cls.train_step, []

        def timed_step(self):                              # pass-through: times the reference's own step
            t0 = time.time()
            orig_step(self)
            steps.append(time.time() - t0)
        cls.train_step = timed_step
        try:
            got, recs, checksum, dt = ref_stubs.run_c1(
                lambda tsv, d, extra: synth_c1.als_yaml(tsv, d, model, epochs, block, extra=extra))
        finally:
            cls.train_step = orig_step
        assert len(recs) == epochs, list(recs)            # one file per evaluated epoch, `_it=<epoch>`
        name, rec = list(recs.items())[-1]
        p = model.lower()
        out["checksum"] = np.uint64(checksum)
        out.update({f"{p}_epochs": epochs, f"{p}_test_metrics": np.array(got), f"{p}_rec_file": name,
                    f"{p}_rec_files": np.array(list(recs)), f"{p}_reference_seconds": dt,
                    f"{p}_reference_step_seconds": np.array(steps)})
        out.update({f"{p}_{k}": v for k, v in ref_stubs.first_users(rec).items()})
        print(f"{model} c1: per-epoch metrics {got}, train_step {steps} s, run {dt:.0f} s, {name}", flush=True)
    np.savez_compressed(os.path.join(GOLD, "als_c1.npz"), **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    args = ap.parse_args()
    _scipy_dense_alias()
    synthetic(ref_stubs.REF)
    if not args.skip_c1:
        c1_runs()


if __name__ == "__main__":
    main()
