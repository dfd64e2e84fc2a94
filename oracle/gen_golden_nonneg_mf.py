#!/usr/bin/env python
"""Mint the NonNegMF goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/nonneg_mf_cases.npz
      the reference's own `NonNegMFModel` (latent_factor_models/NonNegMF/non_negative_matrix_factorization_model.py),
      imported by file path, trained for EPOCHS epochs on small synthetic rating sets.  The cases cover ratings 1-5 with
      explicit 0 ratings, half stars, F = 10, 33 and 1, non-default lr and reg, every user's dict order shuffled, a
      one-rating user, a one-rating item and a user with fewer than k candidates.  Recorded per case: the dict-order CSR
      (indptr, items, ratings), mu, the tables P, Q, bu and bi at the start and after every epoch, and the last epoch's
      `get_user_recs` (items, values).  Before saving, oracle/nonneg_mf.py must reproduce every table of every epoch bit
      for bit, and every table must be finite.
  tests/golden/nonneg_mf_c1.npz
      elliot.run.run_experiment on synth_c1.nonneg_mf_yaml over the C1 synthetic file (oracle/ref_stubs.py harness): the
      test metrics of every epoch, the names of the rec files (one per epoch), the last one's first 400 users' lists, the
      dataset checksum, the wall time of the run and of every train_step.

The reference allocates its biases and its four per-epoch accumulators with `np.empty` (model.py:37-38, 45-48) under the
comment "(re)initialize nums and denominators to zero", and then adds to them: run as written it reads whatever memory
the allocator hands back.  Both goldens therefore pin the evident intent: the `np` name of the reference model's module
is replaced by a shim whose `empty` is `zeros` and which is numpy otherwise.  No line of the reference is changed.  For
every call, the shim also takes the np.empty array the reference asked for and counts its non-zero elements; the script
prints the counts of the C1 run, i.e. what the reference would have read in the process that mints.

    python oracle/gen_golden_nonneg_mf.py [--skip-c1] [--skip-cases]
"""
import argparse
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import nonneg_mf as onm, ref_stubs  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
MODEL = "elliot/recommender/latent_factor_models/NonNegMF/non_negative_matrix_factorization_model.py"
TOPK = 10
EPOCHS = 4
# name: (users, items, mean items per user, rating levels, factors, lr, reg, seed)
CASES = {
    "stars": (90, 120, 14, np.arange(1.0, 6.0), 10, 0.001, 0.1, 42),
    "half_stars": (70, 97, 16, np.arange(1.0, 11.0) / 2, 33, 0.004, 0.03, 7),
    "one_factor": (50, 64, 12, np.arange(1.0, 6.0), 1, 0.02, 0.25, 3),
}


class NumpyZeroEmpty:
    """numpy, except that `empty` is `zeros`: installed as the reference model module's `np`.  `seen` lists, per call,
    (shape, non-zero elements, size) of the np.empty array the call would have returned."""

    def __init__(self):
        self.seen = []

    def empty(self, *args, **kwargs):
        garbage = np.empty(*args, **kwargs)
        self.seen.append((garbage.shape, int(np.count_nonzero(garbage)), garbage.size))
        return np.zeros(*args, **kwargs)

    def __getattr__(self, name):
        return getattr(np, name)


class _Data:
    """The DataSet fields the reference's NonNegMFModel reads; public ids == private ids."""

    def __init__(self, rows, n_items):
        self.num_users, self.num_items = len(rows), n_items
        self.users, self.items = list(range(self.num_users)), list(range(n_items))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}
        self.i_train_dict = self.train_dict = {u: dict(r) for u, r in enumerate(rows)}
        u = np.array([a for a, r in enumerate(rows) for _ in r])
        i = np.array([b for r in rows for b, _ in r])
        v = np.array([c for r in rows for _, c in r])
        shape = (self.num_users, n_items)
        self.sp_i_train = sp.csr_matrix((np.ones_like(u), (u, i)), dtype="float32", shape=shape)
        self.sp_i_train_ratings = sp.csr_matrix((v, (u, i)), dtype="float32", shape=shape)


def ratings(seed, U, I, mean_items, levels):
    """Per user a list of (item, rating) in a shuffled (dict) order: items drawn by a skewed popularity, user 0 with one
    item, user 1 with all but 6 of the items 0..I-2 (with item I-1, fewer than k candidates), item I-1 rated by user 2
    alone, every item rated at least once, and about 2 % explicit 0 ratings."""
    g = np.random.default_rng(seed)
    pop = (1.0 / np.arange(1, I) ** 0.9)[g.permutation(I - 1)]
    pop /= pop.sum()
    counts = np.clip(g.lognormal(np.log(mean_items), 0.6, U), 2, (I - 1) // 2).astype(np.int64)
    sets = [set(g.choice(I - 1, size=int(counts[u]), replace=False, p=pop).tolist()) for u in range(U)]
    sets[0] = {int(g.integers(I - 1))}
    sets[1] = set(range(I - 1)) - set(g.choice(I - 1, size=6, replace=False).tolist())
    for i in set(range(I - 1)) - set().union(*sets):
        sets[int(g.integers(3, U))].add(i)
    sets[2].add(I - 1)
    rows = []
    for s in sets:
        it = g.permutation(sorted(s))
        r = g.choice(levels, size=it.size)
        r[g.random(it.size) < 0.02] = 0.0
        rows.append([(int(a), float(b)) for a, b in zip(it, r)])
    return rows


def csr_of(rows):
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    items = np.array([i for r in rows for i, _ in r], np.int64)
    vals = np.array([v for r in rows for _, v in r], np.float64)
    return indptr, items, vals


def same(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.uint64), np.asarray(b, np.float64).view(np.uint64))


def synthetic(ref_root):
    mod = ref_stubs.load(os.path.join(ref_root, MODEL), "ref_nonneg_mf_model")
    mod.np = NumpyZeroEmpty()
    out = {"cases": np.array(list(CASES)), "topk": TOPK, "epochs": EPOCHS}
    for c, (name, (U, I, mean_items, levels, F, lr, reg, seed)) in enumerate(CASES.items()):
        rows = ratings(c + 1, U, I, mean_items, levels)
        data = _Data(rows, I)
        mu = np.mean(data.sp_i_train_ratings)                 # the reference's own expression (non_negative_matrix_factorization.py)
        assert isinstance(mu, np.float32), type(mu)
        m = mod.NonNegMFModel(data, U, I, mu, F, reg, lr, random_seed=seed)
        indptr, items, vals = csr_of(rows)
        P, Q = onm.init_tables(seed, U, I, F)
        bu, bi = np.zeros(U), np.zeros(I)
        tabs = {"P": [m._user_embeddings.copy()], "Q": [m._item_embeddings.copy()], "bu": [m._user_bias.copy()],
                "bi": [m._item_bias.copy()]}
        for e in range(EPOCHS):
            m.train_step()
            P, Q, _, _ = onm.epoch(P, Q, bu, bi, mu, indptr, items, vals, lr, reg)
            for key, ref, ours in (("P", m._user_embeddings, P), ("Q", m._item_embeddings, Q), ("bu", m._user_bias, bu),
                                   ("bi", m._item_bias, bi)):
                assert np.isfinite(ref).all(), (name, e, key)
                assert same(ref, ours), (name, e, key)
                tabs[key].append(ref.copy())
        cand = np.ones((U, I), bool)
        cand[onm.row_of(indptr), items] = False
        ti = np.full((U, TOPK), -1, np.int64)
        tv = np.full((U, TOPK), -np.inf)
        for u in range(U):
            recs = m.get_user_recs(u, cand, TOPK)
            ti[u, :len(recs)] = [int(i) for i, _ in recs]
            tv[u, :len(recs)] = [float(v) for _, v in recs]
        out.update({f"{name}_shape": np.array([U, I, F]), f"{name}_lr": lr, f"{name}_reg": reg, f"{name}_seed": seed,
                    f"{name}_mu": np.float64(mu), f"{name}_indptr": indptr, f"{name}_items": items.astype(np.int32),
                    f"{name}_ratings": vals, f"{name}_topk_idx": ti, f"{name}_topk_val": tv})
        out.update({f"{name}_{key}": np.stack(v) for key, v in tabs.items()})
        print(f"{name}: {U} x {I}, F={F}, {items.size} ratings, max|P| after {EPOCHS} epochs "
              f"{np.abs(tabs['P'][-1]).max():.3g}", flush=True)
    np.savez_compressed(os.path.join(GOLD, "nonneg_mf_cases.npz"), **out)


def c1_run():
    ref_stubs.install()
    from elliot.recommender.latent_factor_models.NonNegMF import non_negative_matrix_factorization_model as mod
    shim = mod.np = NumpyZeroEmpty()
    epoch_seconds = []
    train_step = mod.NonNegMFModel.train_step

    def timed_train_step(self):                          # pass-through: records each epoch's wall time
        t0 = time.time()
        train_step(self)
        epoch_seconds.append(time.time() - t0)
    mod.NonNegMFModel.train_step = timed_train_step
    got, recs, checksum, dt = ref_stubs.run_c1(lambda tsv, d, extra: synth_c1.nonneg_mf_yaml(tsv, d, extra=extra))
    assert len(got) == 10 and len(recs) == 10, (got, list(recs))
    name = [f for f in recs if f.endswith(f"_it={len(got)}.tsv")]
    assert len(name) == 1, list(recs)
    name = name[0]
    out = {"metrics": np.array(ref_stubs.METRICS), "test_metrics": np.array(got), "rec_files": np.array(list(recs)),
           "rec_file": name, "checksum": np.uint64(checksum), "reference_seconds": dt,
           "reference_epoch_seconds": np.array(epoch_seconds)}
    out.update(ref_stubs.first_users(recs[name]))
    np.savez_compressed(os.path.join(GOLD, "nonneg_mf_c1.npz"), **out)
    print(f"c1: last metrics {got[-1]}, run {dt:.1f} s, {name}", flush=True)
    for shape, nz, size in shim.seen[:6]:
        print(f"np.empty{shape} in the C1 run: {nz} of {size} elements non-zero", flush=True)


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
