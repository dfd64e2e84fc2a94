"""Time SVD++ and FunkSVD through the model's own code (recommender/rating_mf.py's RatingMFModel) at the C1 shape
(synth_c1's 6 040 x 3 706 file) and the ML-20M shape (benchlib's seeded 138 493 x 26 744 matrix), factors 10 (the
reference's default).  80 % of each data set's ratings are the train set, the other 20 % the relevant test items of the
pair pass.  Per model, shape and batch size (512, 8 192): one epoch of `transactions` samples split into its phases
(sampler, implicit mean, fused step, Adam), the recommendation pass (top-10 of every user, with the implicit means) and
the pair pass (the score of every test item), each the median of benchlib.repeat over `--iters` runs after one warm-up.
The reference's TensorFlow arm is not timed: TensorFlow is not installed where this runs.  Prints one JSON line per
model, shape and batch size, with the card, its power limit and clocks.

    python tools/rating_mf_bench.py [--iters 3] [--out results/rating_mf_bench.json]
"""
import argparse
import json
import os

import numpy as np
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.rating_mf import RatingMFModel

F = 10


def split(u, i, r, n_users, seed=0):
    """(train CSR with ratings aligned, item-sorted relevant CSR) on the device: a seeded 80 / 20 split."""
    g = np.random.default_rng(seed)
    test = g.random(u.size) < 0.2
    tu, ti, tr = u[~test], i[~test], r[~test]
    o = np.lexsort((ti, tu))
    mp, mi = bl.train_mask(tu, ti, n_users)
    rel_u, rel_i = u[test], i[test]
    rp = np.zeros(n_users + 1, np.int64)
    np.cumsum(np.bincount(rel_u, minlength=n_users), out=rp[1:])
    rel = bl.upload(rp, bl.DEV, torch.int64), bl.upload(rel_i[np.lexsort((rel_i, rel_u))], bl.DEV, torch.int32)
    return (mp, mi, bl.upload(tr[o], bl.DEV, torch.float32)), rel, int(tu.size)


def epoch(m, implicit, csr, n_users, n_items, T, B, filt):
    mp, mi, rat = csr

    def run(mark):
        if implicit:
            u, i, y = ops.rated_sample_philox(n_users, n_items, mp, mi, rat, T, 42)
        else:
            u, i, y = ops.pointwise_sample_philox(n_users, n_items, mp, mi, T, 42, filter=filt)
        mark("sampler")
        for s in range(0, T, B):
            e = min(s + B, T)
            batch = (u[s:e], i[s:e], y[s:e])
            m._loss.zero_()
            z = None
            if implicit:
                z = m.batch_means(batch[0])
                mark("implicit_mean")
            m.grads(batch, z)
            mark("step")
            m.adam()
            mark("adam")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = bl.card()
    lines = []
    for shape, make in (("C1", bl.c1_matrix), ("ML-20M", bl.ml20m_matrix)):
        u, i, r, n_users, n_items = make()
        csr, (rp, ri), T = split(u, i, r, n_users)
        filt = ops.bloom_build(csr[0], csr[1], n_users)
        for implicit, name in ((True, "SVDpp"), (False, "FunkSVD")):
            m = RatingMFModel(n_users, n_items, F, 1e-3, 42, csr[0], csr[1], implicit, bl.DEV)
            passes = bl.repeat(lambda mark: (m.topk(10, csr[0], csr[1]), mark("recommend_k10"),
                                             m.pair_scores(rp, ri, csr[0], csr[1]), mark("pair_pass")), args.iters)
            for B in (512, 8192):
                t = bl.repeat(epoch(m, implicit, csr, n_users, n_items, T, B, filt), args.iters)
                rec = {"model": name, "shape": shape, "users": n_users, "items": n_items, "train": T, "factors": F,
                       "batch": B, "steps": -(-T // B), "epoch_ms": round(sum(t.values()), 2),
                       **{f"{k}_ms": round(v, 2) for k, v in t.items()},
                       **{f"{k}_ms": round(v, 3) for k, v in passes.items()}, "relevant": int(ri.numel()),
                       "reference": "not timed (TensorFlow is not installed)", "iters": args.iters, **card}
                print(json.dumps(rec), flush=True)
                lines.append(rec)
            del m
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
