#!/usr/bin/env python
"""Mint the ItemKNN / UserKNN goldens from the UNMODIFIED reference (build container only; the tests read the .npz):

  tests/golden/{itemknn,userknn}_{tiny,small}.npz
      the reference's `Similarity` classes (knn/item_knn/item_knn_similarity.py, knn/user_knn/user_knn_similarity.py),
      imported by file path, on synthetic matrices: ratings 1-5, implicit ones and half stars; cosine and dot; a user and
      an item without ratings; (small) a duplicated item, so exact ties exist.  Recorded per case: the reference's fp32/fp64
      preds, its neighbour lists (the arguments of its W constructor, through a pass-through wrapper of
      `sparse.csc_matrix`) and its top-k lists from `get_user_recs`.
  tests/golden/itemknn_c1.npz
      elliot.run.run_experiment on config_files/sample_hello_world.yml's ItemKNN block (neighbors 50, cosine, save_recs)
      over the C1 synthetic file of elliot_b200/synth_c1.py (oracle/ref_stubs.py harness, as gen_golden_c1.py): test
      metrics, the stored rec file's name and the lists of its first 400 users, the dataset checksum, the wall time.

Every synthetic case is also checked against the fp64 restatement oracle/knn.py: its preds over the reference's own
neighbour lists are within 1e-5 relative of the reference's.

    python oracle/gen_golden_knn.py [--skip-c1]
"""
import argparse
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import knn as oknn, ref_stubs  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
TOPK = 10


class _Data:
    """The DataSet fields the reference's Similarity classes read; public ids == private ids."""

    def __init__(self, R):
        U, I = R.shape
        m = sp.csr_matrix(R.astype(np.float32))
        self.sp_i_train_ratings = m
        self.sp_i_train = sp.csr_matrix((np.ones(m.nnz, np.float32), m.indices, m.indptr), shape=m.shape)
        self.users, self.items = list(range(U)), list(range(I))
        self.private_users = self.public_users = {u: u for u in self.users}
        self.private_items = self.public_items = {i: i for i in self.items}
        self.train_dict = {u: {int(i): float(R[u, i]) for i in np.flatnonzero(R[u])} for u in self.users}
        self.transactions = m.nnz


def _matrix(g, U, I, kind, dup):
    R = np.zeros((U, I))
    dens = g.random((U, I)) < 0.3
    if kind == "half":
        vals = g.integers(1, 11, (U, I)) / 2.0
    else:
        vals = g.integers(1, 6, (U, I)).astype(np.float64)
    R[dens] = vals[dens]
    R[U - 2, :] = 0                                      # a user without ratings
    R[:, I - 2] = 0                                      # an item without ratings
    if dup:
        R[:, 1] = R[:, 0]                                # a duplicated item: exact ties in every similarity
        R[3, :] = R[2, :]                                # a duplicated user
    return R


def _reference_case(mod, R, over, k_nn, sim, implicit):
    data = _Data(R)
    made = {}
    real_csc = mod.sparse.csc_matrix

    class _Sparse:                                       # pass-through: records W's arguments, builds it unchanged
        def __getattr__(self, a):
            return getattr(sp, a)

        @staticmethod
        def csc_matrix(arg, **kw):
            made["w"] = arg
            return real_csc(arg, **kw)
    mod.sparse = _Sparse()
    try:
        s = mod.Similarity(data=data, num_neighbors=k_nn, similarity=sim, implicit=implicit)
        s.initialize()
    finally:
        mod.sparse = sp
    vals, rows, ptr = (np.asarray(a) for a in made["w"])
    n = len(ptr) - 1
    idx = np.full((n, k_nn), -1, np.int32)
    val = np.zeros((n, k_nn), np.float32)
    for c in range(n):
        seg = slice(ptr[c], ptr[c + 1])
        o = np.argsort(-vals[seg], kind="stable")
        m = ptr[c + 1] - ptr[c]
        idx[c, :m], val[c, :m] = rows[seg][o], vals[seg][o]
    preds = np.array(s._preds, dtype=np.float64)
    mask = data.sp_i_train.toarray() == 0
    ti = np.full((R.shape[0], TOPK), -1, np.int64)
    tv = np.full((R.shape[0], TOPK), -np.inf)
    for u in data.users:
        recs = s.get_user_recs(u, mask, TOPK)
        ti[u, :len(recs)] = [int(i) for i, _ in recs]
        tv[u, :len(recs)] = [float(v) for _, v in recs]
    return idx, val, preds, ti, tv


def synthetic(ref_root):
    mods = {"items": ref_stubs.load(os.path.join(ref_root, "elliot/recommender/knn/item_knn/item_knn_similarity.py"), "ref_item_knn"),
            "users": ref_stubs.load(os.path.join(ref_root, "elliot/recommender/knn/user_knn/user_knn_similarity.py"), "ref_user_knn")}
    sizes = {"tiny": (12, 9, 3, False), "small": (150, 80, 10, True)}
    for over, model in (("items", "itemknn"), ("users", "userknn")):
        for size, (U, I, k_nn, dup) in sizes.items():
            out = {"k_nn": k_nn, "topk": TOPK, "over": over}
            g = np.random.default_rng(7 if size == "tiny" else 11)
            for kind in ("int", "implicit", "half"):
                R = _matrix(g, U, I, kind, dup)
                Ru = (R != 0).astype(np.float64) if kind == "implicit" else R
                for sim in ("cosine", "dot"):
                    tag = f"{kind}_{sim}"
                    idx, val, P, ti, tv = _reference_case(mods[over], R, over, k_nn, sim, kind == "implicit")
                    # on the reference's own lists: exact ties at rank k_nn may be broken either way (np.argsort)
                    P_or = oknn.preds(Ru, idx, val, over)
                    scale = np.abs(P).max() or 1.0
                    err = np.abs(P_or - P).max() / scale
                    assert err < 1e-5, (model, size, tag, err)
                    out.update({f"{tag}_R": R, f"{tag}_nbr_idx": idx, f"{tag}_nbr_val": val, f"{tag}_preds": P,
                                f"{tag}_topk_idx": ti, f"{tag}_topk_val": tv})
                    print(f"{model}_{size} {tag}: oracle preds within {err:.1e} relative", flush=True)
            np.savez_compressed(os.path.join(GOLD, f"{model}_{size}.npz"), **out)


def hello_world_c1():
    got, recs, checksum, dt = ref_stubs.run_c1(synth_c1.hello_world_yaml)
    assert len(recs) == 1, list(recs)
    (name, rec), = recs.items()
    np.savez_compressed(os.path.join(GOLD, "itemknn_c1.npz"), metrics=np.array(ref_stubs.METRICS),
                        test_metrics=np.array(got[-1]), rec_file=name, checksum=np.uint64(checksum), reference_seconds=dt,
                        **ref_stubs.first_users(rec))
    print(f"itemknn_c1: metrics {dict(zip(ref_stubs.METRICS, got[-1]))}, reference run {dt:.0f} s, {name}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-c1", action="store_true")
    args = ap.parse_args()
    synthetic(ref_stubs.REF)
    if not args.skip_c1:
        hello_world_c1()


if __name__ == "__main__":
    main()
