#!/usr/bin/env python
"""iALS per-epoch phase timings on one GPU; prints one JSON line.

Per data set and factor count d, ALSModel.train_step (elliot_b200/recommender/als.py, iALS order) and the masked top-10
of every user (eb_score_topk_f64) are timed through the model's phase marks (tools/benchlib.py): Gram Y^T Y and X^T X
(eb_gram_f64, both summed), the user half and the item half (eb_als_solve_f64) and the top-10.  WRMF runs the same
kernels (its two Grams are taken before the user half), so it is not timed separately.  One epoch warms up, then
--epochs epochs are timed and the median is reported.  d <= eb_als_small_d_max() (32) runs the one-row-per-warp mapping,
larger d the one-row-per-CTA mapping: d = 10 and d = 64 / 200 time both sides of the threshold.

Rates are counted from shapes: a half costs nnz d^2 fp64 FLOP for the rank-k updates and n_rows d^3 / 3 for the Cholesky
factorisations (the right-hand sides and triangular solves, 2 nnz d + 2 n_rows d^2, are left out); its bytes are the
gathered rows (8 nnz d), the indices and weights (20 nnz) and the written rows (8 n_rows d).  The lower bound on a half's
time is the larger of FLOP / 67 TFLOP/s (the H100 SXM data-sheet fp64 tensor-core peak, at 700 W; a data-sheet figure,
not one reached) and bytes / 3.35 TB/s (data-sheet HBM3 bandwidth); `bound` names the larger.

The reference's per-epoch host time comes from tests/golden/als_c1.npz: the reference's own iALS train_step at C1 shape,
d = 10, on one host core, timed when the golden was minted, not in this run.

Data sets (benchlib, binarised as sp_i_train is): C1 = the (user, item) pairs of elliot_b200/synth_c1.py's file
(6 040 x 3 706, ~1.0 M entries, no test split); ML-20M-shaped = 138 493 x 26 744, ~18.4 M entries.

    python tools/als_bench.py [--skip-ml20m] [--epochs N]
"""
import argparse
import json
import os

import numpy as np
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.als import ALSModel

PEAK_FP64_TC = 67e12
PEAK_HBM = 3.35e12


def _half_cost(nnz, rows, d):
    flops = nnz * d * d + rows * d ** 3 / 3.0
    nbytes = 8.0 * nnz * d + 20.0 * nnz + 8.0 * rows * d
    return flops, nbytes


def run(data, mask, d, epochs):
    np.random.seed(42)
    m = ALSModel("iALS", d, data, 1.0, 0.1, 1.0, "linear", bl.DEV)

    def epoch(mark):
        m.train_step(mark)
        m.topk(10, *mask)
        mark("score_top10")
    t = bl.repeat(epoch, epochs, seconds=True)
    t["epoch_train"] = t["gram"] + t["user_half"] + t["item_half"]
    nnz = int(data.sp_i_train.nnz)
    t["mapping"] = "warp_per_row" if d <= ops.als_small_d_max() else "cta_per_row"
    for half, rows in (("user_half", data.num_users), ("item_half", int(m.items[4].numel()))):
        fl, by = _half_cost(nnz, rows, d)
        t[f"{half}_tflops"] = fl / t[half] / 1e12
        t[f"{half}_gbytes_per_s"] = by / t[half] / 1e9
        t[f"{half}_bytes"] = by
        fl_t, by_t = fl / PEAK_FP64_TC, by / PEAK_HBM
        t[f"{half}_bound"] = "fp64 tensor-core compute" if fl_t >= by_t else "HBM bandwidth"
        t[f"{half}_share_of_bound"] = max(fl_t, by_t) / t[half]
    assert torch.isfinite(m.X).all() and torch.isfinite(m.Y).all()
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--epochs", type=int, default=2)
    args = ap.parse_args()
    out = bl.card()
    sets = {"c1": (bl.c1_matrix, (10, 64))}
    if not args.skip_ml20m:
        sets["ml20m_shape"] = (bl.ml20m_matrix, (10, 64, 200))
    for name, (make, ds) in sets.items():
        u, i, r, U, I = make()
        data, mask = bl.Data(u, i, r, U, I), bl.train_mask(u, i, U)
        out[name] = {"users": U, "items": I, "entries": int(len(u))}
        for d in ds:
            out[name][f"d{d}"] = run(data, mask, d, args.epochs)
            torch.cuda.empty_cache()
    g = np.load(os.path.join(bl.ROOT, "tests", "golden", "als_c1.npz"))
    out["reference_c1_ials_d10_epoch_seconds"] = {
        "value": float(np.mean(g["ials_reference_step_seconds"])),
        "note": "the reference's iALS train_step on one host core, timed when the golden was minted, not in this run"}
    out["reference_c1_wrmf_d10_epoch_seconds"] = {
        "value": float(np.mean(g["wrmf_reference_step_seconds"])),
        "note": "the reference's WRMF train_step on one host core, timed when the golden was minted, not in this run"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
