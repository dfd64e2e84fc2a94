#!/usr/bin/env python
"""Mint the SlopeOne goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/slope_one_cases.npz
      the reference's own `SlopeOneModel` (algebric/slope_one/slope_one_model.py), imported by file path, on small
      synthetic rating sets with at least 2 048 items each: its `freq` and `dev` are np.empty, which comes back as fresh
      zero pages only from 32 MiB up (glibc's largest mmap threshold), so smaller catalogues would add heap garbage.
      Every user's dict order is shuffled.  The cases cover ratings 1-5 with skewed popularity, half stars, all ratings
      equal (every score is the user's mean: a top-k of ties only), item counts that are not multiples of 8, a cold item,
      a one-item user, a user with fewer than k candidates and explicit 0 ratings.  Recorded per case: the dict-order
      CSR (indptr, items, ratings), the user means, the CRC and a few rows of `dev`, and `get_user_recs` (items, values).
      Before saving, the reference's `freq`, `dev` and `user_mean` are checked bit for bit against oracle/slope_one.py,
      and the number of (user, item) scores that differ between the dict-order and the sorted-order sums is recorded
      (it must not be 0 unless every rating is equal).
  tests/golden/slope_one_c1.npz
      elliot.run.run_experiment on synth_c1.slope_one_yaml over the C1 synthetic file (oracle/ref_stubs.py harness): the
      test metrics, the rec file's name and its first 400 users' lists, the dataset checksum and the wall time.

    python oracle/gen_golden_slope_one.py [--skip-c1] [--skip-cases]
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs, slope_one as oso  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 10
DEV_ROWS = 4                    # rows of `dev` recorded per case (besides its CRC)
# name: (users, items, mean items per user, rating levels)
CASES = {
    "stars": (200, 2050, 24, np.arange(1.0, 6.0)),
    "half_stars": (160, 2048, 28, np.arange(1.0, 11.0) / 2),
    "all_equal": (120, 2049, 20, np.array([4.0])),
}


class _Data:
    """The DataSet fields the reference's SlopeOneModel reads; public ids == private ids."""

    def __init__(self, rows, n_items):
        self.num_users, self.num_items = len(rows), n_items
        self.users, self.items = list(range(self.num_users)), list(range(n_items))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}
        self.i_train_dict = self.train_dict = {u: dict(r) for u, r in enumerate(rows)}


def ratings(seed, U, I, mean_items, levels):
    """Per user a list of (item, rating) in a shuffled (dict) order: items drawn by a skewed popularity, item I - 1 cold,
    user 0 with one item, user 1 with all but 6 warm items (fewer than k candidates), and a few explicit 0 ratings
    when the levels are not all equal."""
    g = np.random.default_rng(seed)
    pop = (1.0 / np.arange(1, I) ** 0.9)[g.permutation(I - 1)]
    pop /= pop.sum()
    counts = np.clip(g.lognormal(np.log(mean_items), 0.6, U), 2, 8 * mean_items).astype(np.int64)
    counts[0] = 1
    counts[1] = I - 1 - 6
    rows = []
    for u in range(U):
        it = g.choice(I - 1, size=int(counts[u]), replace=False, p=pop if u != 1 else None)
        r = g.choice(levels, size=it.size)
        if len(levels) > 1:
            r[g.random(it.size) < 0.02] = 0.0
        rows.append([(int(a), float(b)) for a, b in zip(it, r)])
    return rows


def csr_of(rows):
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    items = np.array([i for r in rows for i, _ in r], np.int64)
    vals = np.array([v for r in rows for _, v in r], np.float64)
    return indptr, items, vals


def synthetic(ref_root):
    mod = ref_stubs.load(os.path.join(ref_root, "elliot/recommender/algebric/slope_one/slope_one_model.py"),
                         "ref_slope_one_model")
    out = {"cases": np.array(list(CASES)), "topk": TOPK}
    for c, (name, (U, I, mean_items, levels)) in enumerate(CASES.items()):
        rows = ratings(c + 1, U, I, mean_items, levels)
        data = _Data(rows, I)
        m = mod.SlopeOneModel(data)
        m.initialize()
        indptr, items, vals = csr_of(rows)
        F, E = oso.deviations(indptr, items, vals, I)
        dev = oso.reference_dev(E)
        means = oso.user_means(indptr, vals)
        assert np.array_equal(m.freq, F), name
        assert oso.crc(m.dev) == oso.crc(dev), name
        assert np.array_equal(np.asarray(m.user_mean, np.float64).view(np.uint64), means.view(np.uint64)), name
        P = oso.scores(E, means, indptr, items)
        Ps = oso.scores(E, means, indptr, oso.sorted_rows(indptr, items, vals)[0])
        cand = np.ones((U, I), bool)
        cand[np.repeat(np.arange(U), np.diff(indptr)), items] = False
        n_sensitive = int((cand & (P != Ps)).sum())
        assert n_sensitive > 0 or len(levels) == 1, name
        mask = cand
        ti = np.full((U, TOPK), -1, np.int64)
        tv = np.full((U, TOPK), -np.inf)
        for u in range(U):
            recs = m.get_user_recs(u, mask, TOPK)
            ti[u, :len(recs)] = [int(i) for i, _ in recs]
            tv[u, :len(recs)] = [float(v) for _, v in recs]
            assert np.array_equal(tv[u, :len(recs)], P[u, ti[u, :len(recs)]]), (name, u)
        dev_rows = np.linspace(0, I - 1, DEV_ROWS).astype(np.int64)
        out.update({f"{name}_n_items": I, f"{name}_indptr": indptr, f"{name}_items": items.astype(np.int32),
                    f"{name}_ratings": vals, f"{name}_means": means, f"{name}_dev_crc": np.uint32(oso.crc(m.dev)),
                    f"{name}_dev_rows": dev_rows, f"{name}_dev": m.dev[dev_rows], f"{name}_topk_idx": ti,
                    f"{name}_topk_val": tv, f"{name}_order_sensitive": n_sensitive})
        print(f"{name}: {U} x {I}, {items.size} ratings, {int((F == 0).sum())} pairs without co-ratings, "
              f"{n_sensitive} scores depend on the dict order", flush=True)
    np.savez_compressed(os.path.join(GOLD, "slope_one_cases.npz"), **out)


def c1_run():
    got, recs, checksum, dt = ref_stubs.run_c1(lambda tsv, d, extra: synth_c1.slope_one_yaml(tsv, d, extra=extra))
    assert len(got) == 1 and len(recs) == 1, (got, list(recs))
    name, rec = list(recs.items())[0]
    out = {"metrics": np.array(ref_stubs.METRICS), "test_metrics": np.array(got[0]), "rec_file": name,
           "checksum": np.uint64(checksum), "reference_seconds": dt}
    out.update(ref_stubs.first_users(rec))
    np.savez_compressed(os.path.join(GOLD, "slope_one_c1.npz"), **out)
    print(f"c1: metrics {got[0]}, run {dt:.1f} s, {name}", flush=True)


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
