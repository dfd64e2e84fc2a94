"""Time MF, PMF, FM and LMF through the models' own code (recommender/rating_mf.py's RatingMFModel, recommender/
logistic_mf.py's LMFModel) at the C1 shape (synth_c1's 6 040 x 3 706 file) and the ML-20M shape (benchlib's seeded
138 493 x 26 744 matrix), factors 10.  80 % of each data set's ratings are the train set, the other 20 % the relevant
test items of the pair pass.  Per model, shape and batch size (512, 8 192, and the full batch for LMF): one epoch split
into its phases (sampler, FM's rating-label pass, fused step, optimizer: Keras Adam over every table, or LMF's touched-row
Adagrad), the recommendation pass (top-10 of every user) and the pair pass (the score of every test item), each the median
of benchlib.repeat over `--iters` runs after one warm-up.  An LMF epoch is two passes of `transactions` samples.  Beside
LMF's measured optimizer time the line carries the computed bytes a dense Adagrad pass over Gi and Bi would move per step
and per epoch (read + write of the variable, the accumulator and the gradient): computed, not measured.  The reference's
TensorFlow arm is not timed: TensorFlow is not installed where this runs.  Prints one JSON line per model, shape and
batch size, with the card, its power limit and clocks.

    python tools/pointwise_mf_bench.py [--iters 3] [--out results/pointwise_mf_bench.json]
"""
import argparse
import json
import os

import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.logistic_mf import LMFModel
from elliot_b200.recommender.rating_mf import RatingMFModel
from rating_mf_bench import split

F = 10
CONFIG = {"MF": {"bias": "none"}, "PMF": {"bias": "none", "init": "normal", "head": "sigmoid"},
          "FM": {"bias": "zero", "global_bias": True}}


def epoch(name, m, csr, n_users, n_items, T, B, filt):
    mp, mi, rat = csr
    passes = 2 if name == "LMF" else 1

    def run(mark):
        for p in range(passes):
            u, i, y = ops.pointwise_sample_philox(n_users, n_items, mp, mi, T, 42, first=p * T, filter=filt)
            mark("sampler")
            if name == "FM":
                ops.rating_labels_(mp, mi, rat, u, i, y)
                mark("labels")
            for s in range(0, T, B):
                e = min(s + B, T)
                batch = (u[s:e], i[s:e], y[s:e])
                m._loss.zero_()
                m.grads(batch)
                mark("step")
                if name == "LMF":
                    m.adagrad(batch[1])
                else:
                    m.adam()
                mark("optimizer")
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
        for name in ("MF", "PMF", "FM", "LMF"):
            if name == "LMF":
                m = LMFModel(n_users, n_items, F, 0.1, 0.5, 1e-3, 42, bl.DEV)
            else:
                m = RatingMFModel(n_users, n_items, F, 1e-3, 42, csr[0], csr[1], False, bl.DEV, **CONFIG[name])
            passes = bl.repeat(lambda mark: (m.topk(10, csr[0], csr[1]), mark("recommend_k10"),
                                             m.pair_scores(rp, ri, csr[0], csr[1]), mark("pair_pass")), args.iters)
            for B in (512, 8192) + ((T,) if name == "LMF" else ()):
                t = bl.repeat(epoch(name, m, csr, n_users, n_items, T, B, filt), args.iters)
                steps = -(-T // B) * (2 if name == "LMF" else 1)
                rec = {"model": name, "shape": shape, "users": n_users, "items": n_items, "train": T, "factors": F,
                       "batch": B, "steps": steps, "epoch_ms": round(sum(t.values()), 2),
                       **{f"{k}_ms": round(v, 2) for k, v in t.items()},
                       **{f"{k}_ms": round(v, 3) for k, v in passes.items()}, "relevant": int(ri.numel())}
                if name == "LMF":
                    dense = 6 * 4 * (n_items * m.ld + n_items)                  # var, acc, grad: read + write, fp32
                    rec.update({"dense_adagrad_bytes_per_step": dense, "dense_adagrad_bytes_per_epoch": dense * steps,
                                "dense_adagrad": "computed, not measured"})
                rec.update({"reference": "not timed (TensorFlow is not installed)", "iters": args.iters, **card})
                print(json.dumps(rec), flush=True)
                lines.append(rec)
            del m
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
