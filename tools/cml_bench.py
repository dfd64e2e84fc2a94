"""Time CML through the model's own code (recommender/cml.py's CMLModel) at the C1 shape (synth_c1's 6 040 x 3 706 file)
and the ML-20M shape (benchlib's seeded 138 493 x 26 744 matrix), factors 100 (the reference's default).  Every rating is
a train transaction.  Per shape and batch size (512, 8 192 and `transactions`, the reference's default, whose B x B
loss the reference cannot form): one epoch split into its phases (the sampler, the gradient step, the three Adam calls),
each the median of benchlib.repeat over `--iters` runs after one warm-up; one step at that batch size split by kernel
(terms, the two key sorts, the scatter with its n_a searches, the bias pass with its n'_b searches) by torch.profiler in a
run of its own; and the recommendation pass (top-10 of every user).  The reference's TensorFlow arm is not timed:
TensorFlow is not installed where this runs.  Prints one JSON line per shape and batch size, with the card, its power
limit and clocks.

    python tools/cml_bench.py [--iters 3] [--out results/cml_bench.json]
"""
import argparse
import json
import os

import torch
from torch.profiler import ProfilerActivity, profile

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.cml import CMLModel

F = 100
KERNELS = {"terms": "cml_terms_kernel", "sort": "RadixSort", "scatter_counts": "cml_scatter_kernel",
           "bias_counts": "cml_bias_kernel"}


def epoch(m, sampler, T, B):
    def run(mark):
        tu, ti, tj = sampler.step(T)
        mark("sampler")
        for s in range(0, T, B):
            e = min(s + B, T)
            m.grads((tu[s:e], ti[s:e], tj[s:e]))
            mark("step")
            m.adam()
            mark("adam")
    return run


def kernel_split(m, batch, steps=5):
    """Device milliseconds of one gradient step by kernel group: the kernels of `steps` profiled steps after a warm-up,
    over the number of steps the profile holds (its bias passes; a trace can miss a session's first launches)."""
    m.grads(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            m.grads(batch)
        torch.cuda.synchronize()
    total = {k: 0.0 for k in KERNELS}
    seen = 0
    for ev in prof.key_averages():
        for k, name in KERNELS.items():
            if name in ev.key:
                total[k] += ev.device_time_total / 1e3
                seen += ev.count if k == "bias_counts" else 0
    for t in m.grad.values():
        t.zero_()
    return {k: v / max(seen, 1) for k, v in total.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = bl.card()
    lines = []
    for shape, make in (("C1", bl.c1_matrix), ("ML-20M", bl.ml20m_matrix)):
        u, i, _, n_users, n_items = make()
        indptr, srt = bl.train_mask(u, i, n_users)
        T = int(srt.numel())
        m = CMLModel(F, 1e-3, 1e-3, 1e-3, 0.5, n_users, n_items, 42, bl.DEV)
        sampler = ops.MtSampler(n_users, n_items, indptr, srt, srt, seed=42)     # sorted rows as the set order: timing only
        rec_pass = bl.repeat(lambda mark: (m.topk(10, indptr, srt), mark("recommend_k10")), args.iters)
        for B in (512, 8192, T):
            t = bl.repeat(epoch(m, sampler, T, B), args.iters)
            tu, ti, tj = sampler.step(T)
            split = kernel_split(m, (tu[:B], ti[:B], tj[:B]))
            rec = {"model": "CML", "shape": shape, "users": n_users, "items": n_items, "train": T, "factors": F,
                   "batch": B, "steps": -(-T // B), "epoch_ms": round(sum(t.values()), 2),
                   **{f"{k}_ms": round(v, 2) for k, v in t.items()},
                   **{f"one_step_{k}_ms": round(v, 3) for k, v in split.items()},
                   **{f"{k}_ms": round(v, 3) for k, v in rec_pass.items()},
                   "reference": "not timed (TensorFlow is not installed)", "iters": args.iters, **card}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        del m, sampler
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
