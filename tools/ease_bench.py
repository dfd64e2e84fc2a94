#!/usr/bin/env python
"""EASE^R phase timings on one GPU; prints one JSON line.

Per data set, EASEModel.initialize() (elliot_b200/recommender/ease.py) and the masked top-10 of every user
(eb_dense_score_topk_f32) are timed through the model's phase marks (tools/benchlib.py): Gram (densify + the exact bf16
tensor-core Gram in slabs + the fp64 normal matrix, eb_ease_normal_f64), inverse (eb_inverse_f64), weights
(eb_ease_weights_f32 and the scoring bound) and the top-10.  One run warms up, then --repeat runs are timed and the
median is reported.  The card's name and power limit are read in the same run.

Rates are counted from shapes: the inverse costs 2 n^3 fp64 FLOP (Gauss-Jordan inversion), against 67 TFLOP/s (the H100
SXM data-sheet fp64 tensor-core peak, at 700 W; a data-sheet figure, not one reached); scoring reads 4 nnz n bytes of B
rows (one fp32 row of B per rating), against 3.35 TB/s (data-sheet HBM3 bandwidth).

The reference's C1 seconds come from tests/golden/ease_c1.npz: the whole reference run_experiment of the EASER block on
one host core, timed when the golden was minted, not in this run.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M ratings 1-5, no test
split); ML-20M-shaped = 138 493 x 26 744 with ~18.4 M half-star ratings.

    python tools/ease_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json

import torch

import benchlib as bl
from elliot_b200.recommender.ease import EASEModel

PEAK_FP64_TC = 67e12
PEAK_HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    args = ap.parse_args()
    out = bl.card()
    sets = {"c1": bl.c1_matrix}
    if not args.skip_ml20m:
        sets["ml20m_shape"] = bl.ml20m_matrix
    for name, make in sets.items():
        u, i, r, U, I = make()
        m, mask = EASEModel(bl.Data(u, i, r, U, I), 1e3, bl.DEV), bl.train_mask(u, i, U)
        nnz = int(m.urm[2].numel())

        def run(mark):
            m.initialize(mark)
            m.topk(10, *mask)
            mark("score_top10")
        t = bl.repeat(run, args.repeat, seconds=True)
        assert torch.isfinite(m.B).all()
        t["total"] = sum(t.values())
        t["inverse_tflops"] = 2.0 * I ** 3 / t["inverse"] / 1e12
        t["inverse_share_of_fp64_tc_peak"] = 2.0 * I ** 3 / PEAK_FP64_TC / t["inverse"]
        t["score_b_bytes"] = 4.0 * nnz * I
        t["score_tb_per_s"] = 4.0 * nnz * I / t["score_top10"] / 1e12
        t["score_share_of_hbm_peak"] = 4.0 * nnz * I / PEAK_HBM / t["score_top10"]
        out[name] = {"users": U, "items": I, "ratings": nnz, **t}
        del m
        torch.cuda.empty_cache()
    out["reference_c1_easer_seconds"] = bl.reference_seconds("ease_c1.npz")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
